"""Numpy restatement of kt_op_process_slice (kintinuous_b200/csrc/kt_slice.cu) that predicts every output value, independent of
oracle/kt_slice_oracle.cpp (test infrastructure only):

  * weight cull (alpha >= cull when cull > 0) and the leaf grid exactly as leaf_grid builds it: inv_leaf = float32(1) / leaf,
    min_b / div_b by float32 floor, output slots in ascending leaf index;
  * centroids bit for bit: the kernel sums int64(x * 2^32), which is exact for a float, and rounds float64(sum) * (1 / (n * 2^32))
    to float32 once; colours bit for bit: uint8(int(float32(sum) / float32(n)));
  * the exact k nearest neighbours under the kernel's own key: float32 dx*dx + dy*dy + dz*dz (no FMA, in that order), ranked by
    (key, slot), kk = min(k, n_out, 32) of them; cKDTree proposes candidates, the float32 key ranks them, and a row whose proposal
    cannot be shown complete is asked again with more candidates (at most the whole cloud);
  * normal and curvature in FP64: the covariance about the query point over those neighbours, PCL 1.7.2's analytic eigen33
    (computeRoots / computeRoots2 / smallest eigenvector) restated, the normal flipped towards (0, 0, 0), curvature |lambda0 / trace|;
    NaN for both with fewer than 3 neighbours;
  * the search path the kernel takes for every point (its stop rule simulated on the same leaf grid, with the margin leaf_grid derives
    from the grid's extent), and, wherever the rule stopped, how far the nearest point outside its cube lies: the rule's premise is
    that no such point has a key <= reach^2.  The margin has to absorb the float rounding of the leaf assignment."""
import numpy as np

KNN_MAX, CAND_CAP, R_CAP, R_START = 32, 768, 10, 3
# search paths, in the order the kernel tries them
PATHS = tuple(f"stop{r}" for r in range(R_START, R_CAP + 1)) + ("covers", "overflow", "rcap", "isolated")
P_COVERS, P_OVERFLOW, P_RCAP, P_ISOLATED = (PATHS.index(p) for p in ("covers", "overflow", "rcap", "isolated"))
# overflow: more than CAND_CAP leaves in a cube; rcap: R_CAP reached with kk candidates but the k-th not provably nearest;
# isolated: fewer than kk points within the +-R_CAP cube.  All three end in the kernel's whole-cloud search.


def leaf_grid(pts, weight_cull, leaf):
    """Weight cull + pcl::VoxelGrid as kt_slice.cu computes it.  Returns None for an empty result, else a dict: xyz (float32, n_out x 3,
    ascending leaf index), rgb (uint8, n_out x 3), ijk (int64 leaf coordinates), count (points per leaf), min_b, div_b, leaf, inv_leaf."""
    keep = (pts["a"] >= weight_cull) if weight_cull > 0 else np.ones(len(pts), bool)
    p = pts[keep]
    if len(p) == 0:
        return None
    leaf = np.float32(leaf)
    inv = np.float32(1.0) / leaf
    xyz = np.stack([p["x"], p["y"], p["z"]], -1).astype(np.float32)
    fl = np.floor(xyz * inv)                                                   # float32 product, float32 floor
    min_b = np.floor(xyz.min(0) * inv).astype(np.int64)
    div_b = np.floor(xyz.max(0) * inv).astype(np.int64) - min_b + 1
    ijk = (fl - min_b.astype(np.float32)).astype(np.int64)                     # (int)(floorf(x * inv) - (float)min_b)
    lin = (ijk[:, 2] * div_b[1] + ijk[:, 1]) * div_b[0] + ijk[:, 0]
    uniq, inverse, count = np.unique(lin, return_inverse=True, return_counts=True)
    n_out = len(uniq)
    fixed = np.rint(xyz.astype(np.float64) * 4294967296.0).astype(np.int64)  # exact: a float times 2^32
    sums = np.zeros((n_out, 3), np.int64)
    np.add.at(sums, inverse, fixed)
    cen = (sums.astype(np.float64) * (1.0 / (count.astype(np.float64) * 4294967296.0))[:, None]).astype(np.float32)
    csum = np.zeros((n_out, 3), np.int64)
    np.add.at(csum, inverse, np.stack([p["r"], p["g"], p["b"]], -1).astype(np.int64))
    rgb = (csum.astype(np.float32) / count.astype(np.float32)[:, None]).astype(np.int64).astype(np.uint8)
    out_ijk = np.stack([uniq % div_b[0], (uniq // div_b[0]) % div_b[1], uniq // (div_b[0] * div_b[1])], -1)
    big = np.abs(np.concatenate([xyz.min(0) * inv, xyz.max(0) * inv])).max()
    margin = np.float32(0.001) + np.float32(4) * (np.nextafter(big, np.float32(np.inf)) - big)   # the stop rule's margin, as leaf_grid sets it
    return dict(xyz=cen, rgb=rgb, ijk=out_ijk, count=count, min_b=min_b, div_b=div_b, leaf=leaf, inv_leaf=inv, margin=margin)


def keys32(xyz, q, nb):
    """The kernel's squared distance from points q to points nb (index arrays of one shape), float32, no FMA, x + y then + z."""
    d = xyz[nb] - xyz[q][..., None, :] if nb.ndim == q.ndim + 1 else xyz[nb] - xyz[q]
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def _pack(key, slot):
    """(key, slot) as one uint64 whose integer order is the kernel's (distance, slot) order (key >= 0)."""
    return (key.astype(np.float32).view(np.uint32).astype(np.uint64) << np.uint64(32)) | slot.astype(np.uint64)


def knn(xyz, k):
    """The k smallest (key, slot) of every point over the whole cloud: (slots, keys), each n x min(k, n), ascending."""
    from scipy.spatial import cKDTree
    n = len(xyz)
    k = min(k, n)
    tree = cKDTree(xyz.astype(np.float64))
    slots = np.zeros((n, k), np.int64); keys = np.zeros((n, k), np.float32)
    todo, kq = np.arange(n), min(n, k + 8)
    while len(todo):
        dist, cand = tree.query(xyz[todo].astype(np.float64), k=kq)
        cand = cand.reshape(len(todo), kq)
        packed = np.sort(_pack(keys32(xyz, todo, cand), cand), axis=1)[:, :k]
        s = (packed & np.uint64(0xffffffff)).astype(np.int64)
        kv = (packed >> np.uint64(32)).astype(np.uint32).view(np.float32)
        # every point cKDTree left out is at least dist[:, -1] away in FP64; the float32 key is within 3e-7 of the FP64 square
        ok = np.ones(len(todo), bool) if kq == n else kv[:, -1].astype(np.float64) < dist.reshape(len(todo), kq)[:, -1] ** 2 * (1 - 1e-5)
        slots[todo[ok]] = s[ok]; keys[todo[ok]] = kv[ok]
        todo, kq = todo[~ok], min(n, 4 * kq)
    return slots, keys


def search_paths(g, kk, exact_slots, exact_keys, margin=None):
    """The kernel's search for every output point: r = 3 .. R_CAP over the cube of +-r leaves (clipped to the grid), break on more than
    CAND_CAP candidates, stop when the cube covers the grid or holds kk candidates whose kk-th key is <= reach^2 with
    reach = (r - margin) * leaf (float32; margin: the grid's, unless given).  Returns, per point: the path index; whether a point outside
    the cube it stopped on had a key <= reach^2 (the rule's premise broken); whether that cube missed one of the exact kk nearest; and
    s, the nearest point outside that cube lying r + s leaves away (s capped at 0.5; NaN where the search did not stop on the rule)."""
    from scipy.spatial import cKDTree
    xyz, ijk, div = g["xyz"], g["ijk"], g["div_b"]
    margin = g["margin"] if margin is None else np.float32(margin)
    n = len(xyz)
    tree, ptree = cKDTree(ijk.astype(np.float64)), cKDTree(xyz.astype(np.float64))
    path = np.full(n, -1, np.int64); unsafe = np.zeros(n, bool); wrong = np.zeros(n, bool); slack = np.full(n, np.nan)
    exact_kth = _pack(exact_keys[:, kk - 1], exact_slots[:, kk - 1])
    pend = np.arange(n)
    for r in range(R_START, R_CAP + 1):
        if not len(pend):
            break
        c = ijk[pend]
        covers = ((c - r <= 0) & (c + r >= div - 1)).all(1)
        lists = tree.query_ball_point(ijk[pend].astype(np.float64), r + 0.5, p=np.inf)
        m = np.array([len(li) for li in lists], np.int64)
        cand = np.concatenate([np.asarray(li, np.int64) for li in lists])
        qid = np.repeat(np.arange(len(pend)), m)
        packed = _pack(keys32(xyz, pend[qid], cand), cand)
        order = np.lexsort((packed, qid))
        start = np.concatenate([[0], np.cumsum(m)[:-1]])
        take = np.minimum(kk, m)
        kth = packed[order[start + np.maximum(take, 1) - 1]]
        dk = (kth >> np.uint64(32)).astype(np.uint32).view(np.float32)
        reach = (np.float32(r) - margin) * g["leaf"]
        over = m > CAND_CAP
        stop = ~over & (covers | ((m >= kk) & (dk <= reach * reach)))
        path[pend[over]] = P_OVERFLOW
        path[pend[stop]] = np.where(covers[stop], P_COVERS, PATHS.index(f"stop{r}"))
        wrong[pend[stop]] = kth[stop] != exact_kth[pend[stop]]
        # the premise of the rule, checked directly: every point outside the cube is farther than reach
        ruled = pend[stop & ~covers]
        if len(ruled):
            near = ptree.query_ball_point(xyz[ruled].astype(np.float64), (r + 0.5) * float(g["leaf"]))
            cnt = np.array([len(li) for li in near], np.int64)
            nb = np.concatenate([np.asarray(li, np.int64) for li in near])
            qq = np.repeat(ruled, cnt)
            outside = (np.abs(ijk[nb] - ijk[qq]) > r).any(1)
            key = np.where(outside, keys32(xyz, qq, nb), np.float32(np.inf))
            least = np.full(len(ruled), np.inf, np.float32)
            np.minimum.at(least, np.repeat(np.arange(len(ruled)), cnt), key)
            unsafe[ruled] = least <= reach * reach
            slack[ruled] = np.minimum(np.sqrt(least.astype(np.float64)) / float(g["leaf"]) - r, 0.5)
        if r == R_CAP:
            rest = ~over & ~stop
            path[pend[rest]] = np.where(m[rest] >= kk, P_RCAP, P_ISOLATED)
        pend = pend[~over & ~stop]
    return path, unsafe, wrong, slack


def _roots2(b, c):
    d = np.maximum(b * b - 4.0 * c, 0.0)
    sd = np.sqrt(d)
    return np.stack([np.zeros_like(b), 0.5 * (b - sd), 0.5 * (b + sd)], -1)


def eigen33_smallest(mat):
    """PCL 1.7.2 eigen33 (common/impl/eigen.hpp) in FP64 for a stack of symmetric 3 x 3 matrices (..., 9), row-major: the smallest
    root of the scaled characteristic cubic and the longest cross product of two rows of (A - lambda0 I), normalised."""
    mat = np.asarray(mat, np.float64).reshape(-1, 9)
    scale = np.abs(mat).max(1)
    scale = np.where(scale <= np.finfo(np.float64).tiny, 1.0, scale)
    m = mat / scale[:, None]
    c0 = m[:, 0] * m[:, 4] * m[:, 8] + 2.0 * m[:, 1] * m[:, 2] * m[:, 5] - m[:, 0] * m[:, 5] * m[:, 5] - m[:, 4] * m[:, 2] * m[:, 2] - m[:, 8] * m[:, 1] * m[:, 1]
    c1 = m[:, 0] * m[:, 4] - m[:, 1] * m[:, 1] + m[:, 0] * m[:, 8] - m[:, 2] * m[:, 2] + m[:, 4] * m[:, 8] - m[:, 5] * m[:, 5]
    c2 = m[:, 0] + m[:, 4] + m[:, 8]
    with np.errstate(invalid="ignore"):
        c2_over_3 = c2 * (1.0 / 3.0)
        a_over_3 = np.minimum((c1 - c2 * c2_over_3) * (1.0 / 3.0), 0.0)
        half_b = 0.5 * (c0 + c2_over_3 * (2.0 * c2_over_3 * c2_over_3 - c1))
        q = np.minimum(half_b * half_b + a_over_3 * a_over_3 * a_over_3, 0.0)
        rho = np.sqrt(-a_over_3)
        theta = np.arctan2(np.sqrt(-q), half_b) * (1.0 / 3.0)
        ct, st = np.cos(theta), np.sin(theta)
        s3 = np.sqrt(3.0)
        roots = np.stack([c2_over_3 + 2.0 * rho * ct, c2_over_3 - rho * (ct + s3 * st), c2_over_3 - rho * (ct - s3 * st)], -1)
    # the two conditional swaps of computeRoots (not a sort: it swaps on >=)
    for a, b in ((0, 1), (1, 2)):
        sw = roots[:, a] >= roots[:, b]
        roots[sw, a], roots[sw, b] = roots[sw, b], roots[sw, a].copy()
        if b == 2:
            sw2 = sw & (roots[:, 0] >= roots[:, 1])
            roots[sw2, 0], roots[sw2, 1] = roots[sw2, 1], roots[sw2, 0].copy()
    use2 = (np.abs(c0) < np.finfo(np.float64).eps) | (roots[:, 0] <= 0.0)
    roots[use2] = _roots2(c2[use2], c1[use2])
    ev = roots[:, 0] * scale
    s = m.copy()
    for i in (0, 4, 8):
        s[:, i] -= roots[:, 0]
    r0, r1, r2 = s[:, 0:3], s[:, 3:6], s[:, 6:9]
    vs = np.stack([np.cross(r0, r1), np.cross(r0, r2), np.cross(r1, r2)], 1)
    ls = (vs * vs).sum(2)
    pick = np.where((ls[:, 0] >= ls[:, 1]) & (ls[:, 0] >= ls[:, 2]), 0, np.where(ls[:, 1] >= ls[:, 2], 1, 2))
    v = vs[np.arange(len(vs)), pick]
    with np.errstate(invalid="ignore", divide="ignore"):
        v = v / np.sqrt(ls[np.arange(len(vs)), pick])[:, None]
    return ev, v


def normals(xyz, slots):
    """FP64 normal (flipped towards the origin), curvature and numpy.linalg.eigh eigenvalues of every point's neighbourhood
    (slots: n x kk, the query point's own row first or not); NaN for kk < 3."""
    n, kk = slots.shape
    if kk < 3:
        nan = np.full(n, np.nan)
        return np.stack([nan, nan, nan], -1), nan, np.full((n, 3), np.nan)
    x = xyz.astype(np.float64)
    d = x[slots] - x[:, None, :]                                               # about the query point
    a = np.einsum("nki,nkj->nij", d, d) / kk
    mu = d.mean(1)
    cov = a - mu[:, :, None] * mu[:, None, :]
    ev, v = eigen33_smallest(cov.reshape(n, 9))
    tr = cov[:, 0, 0] + cov[:, 1, 1] + cov[:, 2, 2]
    with np.errstate(invalid="ignore", divide="ignore"):
        curv = np.where(tr != 0.0, np.abs(ev / tr), 0.0)
    flip = (-(x * v).sum(1)) < 0
    v[flip] = -v[flip]
    return v, curv, np.linalg.eigh(cov)[0]


def process_slice(pts, weight_cull, leaf, k=20, margin=None):
    """Everything kt_op_process_slice writes, predicted, plus what the GPU test needs to judge it.  None when the cull keeps nothing.
    margin: simulate the search with this stop-rule margin instead of the grid's."""
    g = leaf_grid(pts, weight_cull, leaf)
    if g is None:
        return None
    xyz = g["xyz"]
    n = len(xyz)
    kk = min(k, n, KNN_MAX)
    slots, keys = knn(xyz, min(kk + 1, n))                                     # one more: the neighbour a wrong search would take instead
    nrm, curv, w = normals(xyz, slots[:, :kk])
    path, unsafe, wrong, slack = search_paths(g, kk, slots, keys, margin)
    return dict(g, kk=kk, slots=slots, keys=keys, normal=nrm, curvature=curv, eig=w, path=path, stop_unsafe=unsafe, stop_wrong=wrong,
                stop_slack=slack)


def unmet(ref, expect, gap_min):
    """What a scene was built for and does not reach: {path name or "ties": least count} over the points whose eigen-gap
    (lambda1 - lambda0) / lambda2 is at least gap_min ("ties": points whose k-th and (k+1)-th keys are equal).  Also returns the mask."""
    kk = ref["kk"]
    w = ref["eig"]
    checked = (w[:, 1] - w[:, 0]) >= gap_min * w[:, 2] if kk >= 3 else np.zeros(len(w), bool)
    taken = np.bincount(ref["path"][checked], minlength=len(PATHS))
    got = {what: int((ref["keys"][:, kk - 1] == ref["keys"][:, kk]).sum()) if what == "ties" else int(taken[PATHS.index(what)]) for what in expect}
    return {what: (got[what], least) for what, least in expect.items() if got[what] < least}, checked
