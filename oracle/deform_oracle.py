"""CPU restatement (numpy / scipy, FP64) of the embedded deformation graph of Kintinuous's backend, the yardstick of kt_deform.cu.

Written from the reference's description (src/backend/DeformationGraph.cpp, Deformation.cpp), not from its code:
  sample_nodes        initialiseGraphPoses (DeformationGraph.cpp:51-86)
  connect_seq         connectGraphSeq (:217-271)
  nearest_node        the binary search of weightVerticesSeq (:454-498), indices clamped to the node range (quirk R2)
  weights             weightVerticesSeq (:441-556)
  residual / jacobian sparseResidual(Cons) / sparseJacobian (:776-988), J as a scipy.sparse matrix in the reference's row order
  optimise            optimiseGraphSparse (:714-774): undamped Gauss-Newton, J^T J solved by scipy.sparse
  apply               computeVertexPosition (:1028-1054)
  pose_constraints    Deformation::addCameraLoop's camera-pose constraints (Deformation.cpp:233-276)

Unknowns: 12 per node, the rotation in column-major order (x[3m+e] = R[e, m]) then the translation.
"""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

K = 4             # Deformation.cpp:469
LOOKBACK = 20     # DeformationGraph.cpp:445
W_REG, W_CON = 10.0, 100.0


def _dist_f32(a, b):
    """||a - b|| in float32, ((dx*dx + dy*dy) + dz*dz), correctly rounded sqrt; a, b broadcast over [..., 3]."""
    d = (np.asarray(a, np.float32) - np.asarray(b, np.float32)).astype(np.float32)
    s = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]).astype(np.float32)
    s = (s + d[..., 2] * d[..., 2]).astype(np.float32)
    return np.sqrt(s, dtype=np.float32)


def sample_nodes(pos, pose_dist):
    """Indices of the positions taken as nodes: the first, then each one more than pose_dist (float) from the last taken."""
    pos = np.asarray(pos, np.float32)
    take = [0] if len(pos) else []
    for i in range(1, len(pos)):
        if _dist_f32(pos[take[-1]], pos[i]) > np.float32(pose_dist):
            take.append(i)
    return np.array(take, np.int64)


def connect_seq(n, k=K):
    """Neighbour lists of the sequential graph, in the reference's order."""
    out = []
    for i in range(n):
        if i < k // 2:
            out.append([m for m in range(k + 1) if m != i])
        elif i < n - k // 2:
            nb = []
            for m in range(k // 2):
                nb += [i - (m + 1), i + (m + 1)]
            out.append(nb)
        else:
            out.append([m for m in range(n - (k + 1), n) if m != i])
    return out


def nearest_node(times, t):
    """The reference's binary search and nearest-in-time choice for one time, with imin / imax clamped to [0, n)."""
    n = len(times)
    t = int(t)
    imin, imax = 0, n - 1
    imid = (imin + imax) // 2
    while imax >= imin:
        imid = (imin + imax) // 2
        if int(times[imid]) < t:
            imin = imid + 1
        elif int(times[imid]) > t:
            imax = imid - 1
        else:
            break
    imin = min(imin, n - 1)
    imax = max(imax, 0)
    da, dm, db = (abs(int(times[i]) - t) for i in (imin, imid, imax))
    if da <= dm and da <= db:
        return imin
    if dm <= da and dm <= db:
        return imid
    return imax


def nearest_nodes(times, ts):
    """nearest_node over an array of times (node times strictly ascending)."""
    times = np.asarray(times, np.uint64)
    ts = np.asarray(ts, np.uint64)
    n = len(times)
    lo = np.searchsorted(times, ts, side="left")
    exact = (lo < n) & (times[np.minimum(lo, n - 1)] == ts)
    a = np.minimum(lo, n - 1)                                            # imin and imax after the search, clamped
    b = np.maximum(lo - 1, 0)
    da = np.where(times[a] > ts, times[a] - ts, ts - times[a])
    db = np.where(times[b] > ts, times[b] - ts, ts - times[b])
    found = np.where(da <= db, a, b)
    return np.where(exact, lo, found).astype(np.int64)


def weights(node_pos, node_times, v, vt, k=K, chunk=200_000):
    """(ids int32 [N, k] ascending, weights float64 [N, k]) of the vertices v (float32 [N, 3]) at times vt."""
    v = np.asarray(v, np.float32).reshape(-1, 3)
    vt = np.asarray(vt, np.uint64).reshape(-1)
    if len(v) > chunk:
        parts = [weights(node_pos, node_times, v[i:i + chunk], vt[i:i + chunk], k, chunk) for i in range(0, len(v), chunk)]
        return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
    node_pos = np.asarray(node_pos, np.float32)
    n = len(node_pos)
    found = nearest_nodes(node_times, vt)
    lo = np.maximum(found - (LOOKBACK - 1), 0)
    cand = lo[:, None] + np.arange(LOOKBACK)[None, :]
    valid = cand < n
    cand_c = np.minimum(cand, n - 1)
    d = _dist_f32(node_pos[cand_c], v[:, None, :])
    d = np.where(valid & ~np.isnan(d), d, np.float32(np.inf))            # a non-finite vertex still takes nodes of its window, by id
    order = np.argsort(d, axis=1, kind="stable")[:, :k + 1]               # by distance, ties by node id
    ids = np.take_along_axis(cand_c, order, axis=1)
    dmax = np.take_along_axis(d, order[:, k:k + 1], axis=1).astype(np.float64)[:, 0]
    g = node_pos[ids[:, :k]].astype(np.float64)
    e = v.astype(np.float64)[:, None, :] - g
    dd = np.sqrt((e[..., 0] * e[..., 0] + e[..., 1] * e[..., 1]) + e[..., 2] * e[..., 2])
    with np.errstate(invalid="ignore"):                                  # inf / inf of a non-finite vertex: equal weights below
        a = 1.0 - dd / dmax[:, None]
        w = a * a
        s = w[:, 0].copy()
        for q in range(1, k):
            s = s + w[:, q]
        w = np.where(s[:, None] > 0, w / np.where(s > 0, s, 1.0)[:, None], 1.0 / k)
    ids = ids[:, :k]
    o = np.argsort(ids, axis=1, kind="stable")
    return np.take_along_axis(ids, o, axis=1).astype(np.int32), np.take_along_axis(w, o, axis=1)


class Graph:
    """The graph, its constraints and the cost of optimiseGraphSparse."""

    def __init__(self, node_pos, con_src, con_dst, con_ids, con_w, k=K):
        self.g = np.asarray(node_pos, np.float32).astype(np.float64)
        self.n = len(self.g)
        self.nbr = connect_seq(self.n, k)
        self.src = np.asarray(con_src, np.float32).astype(np.float64).reshape(-1, 3)
        self.dst = np.asarray(con_dst, np.float64).reshape(-1, 3)
        self.ids = np.asarray(con_ids, np.int64)
        self.w = np.asarray(con_w, np.float64)
        self.m = len(self.src)
        self.n_reg = sum(len(b) for b in self.nbr)
        self.rows = 6 * self.n + 3 * self.n_reg + 3 * self.m

    @staticmethod
    def identity(n):
        x = np.zeros((n, 12))
        x[:, 0] = x[:, 4] = x[:, 8] = 1.0
        return x

    def vertex_positions(self, x, v, ids, w):
        """computeVertexPosition's position for points v [N, 3] (float64) with node ids / weights [N, k]."""
        R = x[:, :9].reshape(-1, 3, 3).transpose(0, 2, 1)                  # column-major -> R[e, m]
        t = x[:, 9:]
        out = np.zeros_like(v)
        for q in range(ids.shape[1]):
            j = ids[:, q]
            out += w[:, q, None] * (np.einsum("nem,nm->ne", R[j], v - self.g[j]) + self.g[j] + t[j])
        return out

    def residual_cons(self, x):
        return ((self.vertex_positions(x, self.src, self.ids, self.w) - self.dst) * np.sqrt(W_CON)).reshape(-1)

    def residual(self, x):
        r = np.zeros(self.rows)
        c0, c1, c2 = x[:, 0:3], x[:, 3:6], x[:, 6:9]
        rot = np.stack([(c0 * c1).sum(1), (c0 * c2).sum(1), (c1 * c2).sum(1),
                        (c0 * c0).sum(1) - 1.0, (c1 * c1).sum(1) - 1.0, (c2 * c2).sum(1) - 1.0], axis=1)
        r[:6 * self.n] = rot.reshape(-1)
        R = x[:, :9].reshape(-1, 3, 3).transpose(0, 2, 1)
        row = 6 * self.n
        for j in range(self.n):
            for nb in self.nbr[j]:
                r[row:row + 3] = (R[j] @ (self.g[nb] - self.g[j]) + self.g[j] + x[j, 9:] - (self.g[nb] + x[nb, 9:])) * np.sqrt(W_REG)
                row += 3
        r[row:] = self.residual_cons(x)
        return r

    def jacobian(self, x):
        rr, cc, vv = [], [], []

        def put(row, col, val):
            rr.append(row); cc.append(col); vv.append(val)
        for j in range(self.n):
            c = 12 * j
            R = x[j, :9]                                                    # column-major: R[e, m] = x[3m + e]
            col = lambda m: R[3 * m:3 * m + 3]
            b = 6 * j
            for e in range(3):
                put(b, c + e, col(1)[e]); put(b, c + 3 + e, col(0)[e])
                put(b + 1, c + e, col(2)[e]); put(b + 1, c + 6 + e, col(0)[e])
                put(b + 2, c + 3 + e, col(2)[e]); put(b + 2, c + 6 + e, col(1)[e])
                put(b + 3, c + e, 2 * col(0)[e]); put(b + 4, c + 3 + e, 2 * col(1)[e]); put(b + 5, c + 6 + e, 2 * col(2)[e])
        row = 6 * self.n
        s = np.sqrt(W_REG)
        for j in range(self.n):
            c = 12 * j
            for nb in self.nbr[j]:
                d = self.g[nb] - self.g[j]
                for e in range(3):
                    for m in range(3):
                        put(row + e, c + 3 * m + e, d[m] * s)
                    put(row + e, c + 9 + e, s)
                    put(row + e, 12 * nb + 9 + e, -s)
                row += 3
        s = np.sqrt(W_CON)
        for l in range(self.m):
            for q in range(self.ids.shape[1]):
                j = self.ids[l, q]; w = self.w[l, q]
                d = (self.src[l] - self.g[j]) * w
                for e in range(3):
                    for m in range(3):
                        put(row + e, 12 * j + 3 * m + e, d[m] * s)
                    put(row + e, 12 * j + 9 + e, w * s)
            row += 3
        return sp.csr_matrix((vv, (rr, cc)), shape=(self.rows, 12 * self.n))

    def band(self):
        """Widest node-id span of any term (regularisation edge or constraint)."""
        b = max(abs(nb - j) for j in range(self.n) for nb in self.nbr[j])
        if self.m:
            b = max(b, int((self.ids.max(1) - self.ids.min(1)).max()))
        return b

    def optimise(self):
        """optimiseGraphSparse: returns (x [n, 12], report dict with the fields of kt_deform_report)."""
        x = self.identity(self.n)
        rep = dict(nodes=self.n, constraints=self.m, band=self.band(), iterations=0, deformed=0, solver_failed=0)
        r = self.residual(x)
        rep["constraint_error"] = float(np.float32(np.linalg.norm(self.residual_cons(x)) / self.m))
        rep["initial_error"] = rep["final_error"] = float(r @ r)
        if rep["constraint_error"] < 0.1:
            return x, rep
        error = last = float(r @ r)
        it = 0
        while it < 10:
            it += 1
            J = self.jacobian(x)
            A = (J.T @ J).tocsc()
            delta = spla.spsolve(A, -(J.T @ r))
            x = x + delta.reshape(self.n, 12)
            r = self.residual(x)
            error = float(r @ r)
            rep["iterations"] = it
            rep["final_error"] = error
            if np.linalg.norm(delta) < 1e-2 or error < 1e-3 or abs(error - last) < 1e-5 * error:
                break
            last = error
        rep["deformed"] = 1
        return x, rep


def apply(node_pos, x, ids, w, pos, nrm):
    """computeVertexPosition for points pos / normals nrm [N, 3]: (positions, normals) in float64; a zero normal stays zero."""
    g = np.asarray(node_pos, np.float32).astype(np.float64)
    R = x[:, :9].reshape(-1, 3, 3).transpose(0, 2, 1)
    Rit = np.linalg.inv(R).transpose(0, 2, 1)
    t = x[:, 9:]
    v = np.asarray(pos, np.float32).astype(np.float64)
    nv = np.asarray(nrm, np.float32).astype(np.float64)
    p = np.zeros_like(v); nn = np.zeros_like(v)
    for q in range(ids.shape[1]):
        j = ids[:, q]
        p += w[:, q, None] * (np.einsum("nem,nm->ne", R[j], v - g[j]) + g[j] + t[j])
        nn += w[:, q, None] * np.einsum("nem,nm->ne", Rit[j], nv)
    l = np.linalg.norm(nn, axis=1, keepdims=True)
    nn = np.where(l > 0, nn / np.where(l > 0, l, 1.0), 0.0)
    return p, nn


def pose_constraints(graph_times, graph_pos, corr_times, corr_pos):
    """(times, sources float32 [m, 3], targets float64 [m, 3]): each corrected pose pulls the tracked camera position at its time
    (the last dense pose with that timestamp) to the corrected one.  KeyError for a timestamp not in the graph."""
    at = {int(t): i for i, t in enumerate(graph_times)}
    idx = [at[int(t)] for t in corr_times]
    return (np.asarray(corr_times, np.uint64), np.asarray(graph_pos, np.float32)[idx],
            np.asarray(corr_pos, np.float64).reshape(-1, 3))


def deform(dense_times, dense_pos, corr_times, corr_pos, node_spacing, verts, normals, vtimes, points=None):
    """The whole of kt_deform_map over one point set: (positions, normals, report, x, node_pos, node_times)."""
    for a in (dense_pos, corr_pos) + (tuple(points[1:]) if points is not None else ()):
        if not np.isfinite(np.asarray(a, np.float64)).all():
            raise ValueError("a position, source or target is not finite")        # kt_deform_map: KT_ERR_INVALID
    take = sample_nodes(dense_pos, node_spacing)
    node_pos = np.asarray(dense_pos, np.float32)[take]
    node_times = np.asarray(dense_times, np.uint64)[take]
    ct, cs, cd = pose_constraints(dense_times, dense_pos, corr_times, corr_pos)
    if points is not None:
        pt, ps, pd = points
        ct = np.concatenate([ct, np.asarray(pt, np.uint64)]); cs = np.concatenate([cs, np.asarray(ps, np.float32)])
        cd = np.concatenate([cd, np.asarray(pd, np.float64)])
    cids, cw = weights(node_pos, node_times, cs, ct)
    x, rep = Graph(node_pos, cs, cd, cids, cw).optimise()
    if not rep["deformed"]:
        return np.asarray(verts, np.float32).astype(np.float64), np.asarray(normals, np.float32).astype(np.float64), rep, x, node_pos, node_times
    ids, w = weights(node_pos, node_times, verts, vtimes)
    p, n = apply(node_pos, x, ids, w, verts, normals)
    return p, n, rep, x, node_pos, node_times


def warp(t_frac, max_deg=2.0, max_shift=(0.05, -0.02, 0.08)):
    """A time-varying rigid correction W(t): rotation about +y by up to max_deg degrees and a translation, both growing linearly with
    t_frac in [0, 1].  Returns (R [N, 3, 3], t [N, 3])."""
    a = np.deg2rad(max_deg) * np.asarray(t_frac, np.float64)
    c, s = np.cos(a), np.sin(a)
    R = np.zeros(a.shape + (3, 3))
    R[..., 0, 0] = c; R[..., 0, 2] = s; R[..., 1, 1] = 1.0; R[..., 2, 0] = -s; R[..., 2, 2] = c
    return R, np.asarray(t_frac, np.float64)[..., None] * np.asarray(max_shift, np.float64)


def synthetic(seed, n_poses, n_verts, step=0.02, radius=3.0, t0=1_000_000, dt=33_333, spread=1.5):
    """A seeded trajectory (a noisy circle of the given radius, one pose per dt microseconds, about `step` metres apart) and map
    vertices near it (float32 positions, unit normals with every 50th zero, times spread over the trajectory and 2 s either side)."""
    rng = np.random.default_rng(seed)
    ang = np.arange(n_poses) * step / radius
    pos = np.stack([radius * np.cos(ang), 0.3 * np.sin(3 * ang), radius * np.sin(ang)], 1) + rng.normal(0, 0.002, (n_poses, 3))
    times = (t0 + dt * np.arange(n_poses)).astype(np.uint64)
    vt = rng.integers(t0 - 2_000_000, t0 + dt * n_poses + 2_000_000, n_verts).astype(np.uint64)
    at = np.clip(np.searchsorted(times, vt), 0, n_poses - 1)
    v = (pos[at] + rng.uniform(-spread, spread, (n_verts, 3))).astype(np.float32)
    nrm = rng.normal(size=(n_verts, 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    nrm[::50] = 0.0
    return times, pos.astype(np.float32), vt, v, nrm.astype(np.float32)
