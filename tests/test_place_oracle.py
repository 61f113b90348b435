"""Place recognition's restatement (oracle/place_oracle.py) and the host logic of kt_place.hpp, without a GPU: SURF's scale and rotation
behaviour, exact ratio matching, the 3-D lookup quirks, PnP against cv2, fitness against a brute-force nearest neighbour, and
kt_place.hpp against the oracle."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from conftest import ROOT
from oracle import place_oracle as PO


@pytest.fixture(scope="module")
def lib():
    out = os.path.join(ROOT, "tests", "cpp", "_build")
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, "libkt_place_host.so")
    src = os.path.join(ROOT, "tests", "cpp", "place_host.cpp")
    hdr = os.path.join(ROOT, "kintinuous_b200", "csrc", "kt_place.hpp")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-std=c++14", "-O2", "-shared", "-fPIC", "-I", os.path.join(ROOT, "kintinuous_b200", "csrc"), "-o", so, src])
    lib = C.CDLL(so)
    lib.kth_motion.restype = C.c_double
    lib.kth_lookup_3d.argtypes = [C.c_float, C.c_float, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lib.kth_throttled.argtypes = [C.c_uint64, C.c_uint64, C.c_double]
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def test_grey_is_cv2():
    import cv2
    rgb = np.random.default_rng(0).integers(0, 256, (97, 131, 3), dtype=np.uint8)
    assert np.array_equal(PO.grey(rgb), cv2.cvtColor(rgb, cv2.COLOR_RGB2GRAY))


@pytest.mark.parametrize("sigma", [3.0, 5.0, 8.0])
def test_blob_found_at_its_scale(sigma):
    n = 200
    y, x = np.mgrid[0:n, 0:n].astype(np.float64)
    img = 230.0 - 200.0 * np.exp(-((x - 101.3) ** 2 + (y - 98.6) ** 2) / (2 * sigma ** 2))
    rgb = np.repeat(np.rint(img)[..., None], 3, -1).astype(np.uint8)
    kp, _ = PO.surf(rgb, max_features=5)
    assert len(kp) >= 1
    k = kp[0]
    assert abs(k[0] - 101.3) < 0.6 and abs(k[1] - 98.6) < 0.6, k
    s = 1.2 * k[2] / 9.0
    assert abs(s - sigma) / sigma < 0.3, (s, sigma)
    assert k[5] == 1                       # a dark blob on a bright ground: Dxx + Dyy > 0


def test_rotation_by_90_degrees():
    from kintinuous_b200 import synth
    # synth's default checker repeats, so its descriptors have look-alikes; cell_texture's random grey cells do not
    R, t = synth.pose(3)
    _, rgb = synth.render_at(R, t, 240, 240, texture=synth.cell_texture)
    kp, desc = PO.surf(rgb, max_features=150)
    rot = np.ascontiguousarray(np.rot90(rgb))               # (x, y) -> (y, W - 1 - x)
    kr, dr = PO.surf(rot, max_features=150)
    W = rgb.shape[1]
    mapped = np.stack([kp[:, 1], W - 1 - kp[:, 0]], 1)
    d = np.linalg.norm(mapped[:, None, :] - kr[None, :, :2], axis=2)
    j = d.argmin(1); close = d[np.arange(len(kp)), j] < 1.0
    assert close.mean() > 0.7, close.mean()
    # box filters on a pixel grid are rotation invariant only approximately: the counterpart must be the nearest descriptor for most (what
    # matching needs), and much nearer than an unrelated one
    D = ((desc[close][:, None, :] - dr[None]) ** 2).sum(2)
    assert (D.argmin(1) == j[close]).mean() > 0.7, (D.argmin(1) == j[close]).mean()
    dd = np.sqrt(D[np.arange(close.sum()), j[close]])
    assert np.median(dd) < 0.35 and np.median(dd) < 0.5 * np.median(np.sqrt(D)), (np.median(dd), np.median(np.sqrt(D)))
    dang = np.angle(np.exp(1j * (kr[j[close], 3] - kp[close, 3] + np.pi / 2)))      # rot90 turns image directions by -90 degrees (y down)
    assert np.median(np.abs(dang)) < np.deg2rad(10)


def test_ratio_matching_is_brute_force():
    rng = np.random.default_rng(3)
    db = rng.standard_normal((200, 64)); q = rng.standard_normal((50, 64))
    q[:20] = db[:20] + 0.05 * rng.standard_normal((20, 64))
    best, d1, d2, ps = PO.match_ratio(db, q)
    for i in range(len(db)):
        dist = ((db[i] - q) ** 2).sum(1)
        o = np.argsort(dist, kind="stable")
        assert best[i] == o[0] and np.isclose(d1[i], dist[o[0]]) and np.isclose(d2[i], dist[o[1]])
        assert ps[i] == (dist[o[0]] < 0.49 * dist[o[1]])
    assert ps[:20].all()


def test_lookup_quirks(lib):
    depth = np.zeros((10, 12), np.uint16); depth[4, 5] = 1500; depth[4, 6] = 10000; depth[4, 7] = 9999; depth[5, 5] = 0
    intr = np.array([100.0, 100.0, 6.0, 5.0], np.float32)
    # z = 10.000 m is dropped (Surf3DTools.h:82: |z - 10| < FLT_EPSILON), 9.999 m kept
    cases = [(5.2, 3.9, True), (5.5, 4.0, False), (4.5, 4.0, False), (5.0, 4.4999, True), (6.0, 4.0, False), (7.1, 4.0, True), (5.0, 5.0, False),
             (-0.4, 4.0, False)]
    for x, y, ok in cases:
        o = PO.lookup_3d(x, y, depth, intr)
        out = np.zeros(3, np.float32)
        got = lib.kth_lookup_3d(x, y, _p(depth), 10, 12, _p(intr), _p(out))
        assert bool(got) == ok == (o is not None), (x, y)
        if ok:
            assert np.array_equal(out, o)


def test_host_logic_equals_oracle(lib):
    rng = np.random.default_rng(11)
    for _ in range(200):
        Rl = Rotation.from_rotvec(rng.normal(0, 0.5, 3)).as_matrix().astype(np.float32)
        Rc = (Rotation.from_rotvec(rng.normal(0, 0.12, 3)).as_matrix() @ Rl).astype(np.float32)
        gl = rng.normal(0, 1, 3).astype(np.float32); gc = (gl + rng.normal(0, 0.1, 3)).astype(np.float32)
        m = lib.kth_motion(_p(Rc), _p(Rl), _p(gc), _p(gl))
        ang = np.linalg.norm(Rotation.from_matrix(Rc.T.astype(np.float64) @ Rl.astype(np.float64)).as_rotvec())
        assert abs(m - 0.5 * (ang + np.linalg.norm(gc.astype(np.float64) - gl))) < 1e-6
        if abs(m - 0.15) > 1e-5:
            assert bool(lib.kth_is_keyframe(_p(Rc), _p(Rl), _p(gc), _p(gl))) == PO.is_keyframe(Rc, Rl, gc, gl)
    for _ in range(200):
        q = int(rng.integers(0, 60)); passes = rng.integers(0, 80, q + 1).astype(np.int32)
        passes[rng.integers(0, q + 1)] = passes.max()                          # ties go to the older keyframe
        assert lib.kth_select_candidate(_p(passes), q, 20, 40) == PO.select_candidate(passes, q, 20, 40)
    n_old, n_new = 300, 120
    best = rng.integers(-1, n_new, n_old).astype(np.int32); d1 = rng.integers(0, 50, n_old).astype(np.float32)     # integer distances: ties
    ps = (rng.random(n_old) < 0.6).astype(np.uint8)
    oi = np.zeros(n_new, np.int32); ni = np.zeros(n_new, np.int32)
    m = lib.kth_unique_matches(_p(best), _p(d1), _p(ps), n_old, n_new, _p(oi), _p(ni))
    eo, en = PO.unique_matches(best, d1, ps, n_new)
    assert np.array_equal(oi[:m], eo) and np.array_equal(ni[:m], en)
    assert lib.kth_throttled(0, 5, 30.0) == 0 and lib.kth_throttled(1_000_000, 31_000_000, 30.0) == 1 and lib.kth_throttled(1_000_000, 31_000_001, 30.0) == 0


def test_match_3d_order_is_the_references(lib):
    # ratio test over ALL features, one match per new feature, THEN the pairs without a 3-D point dropped (Surf3DTools.h:105-176)
    rng = np.random.default_rng(5)
    n_old, n_new = 400, 300
    new = rng.standard_normal((n_new, 64)); new /= np.linalg.norm(new, axis=1, keepdims=True)
    src = rng.integers(0, n_new, n_old)
    old = new[src] + rng.normal(0, 0.08, (n_old, 64)); old /= np.linalg.norm(old, axis=1, keepdims=True)
    for j in range(0, n_new, 7):                                           # look-alike pairs: a weak ratio test where one of them has no depth
        new[j + 1 if j + 1 < n_new else j] = new[j] + 0.01 * rng.standard_normal(64)
    xyz_old = rng.normal(0, 1, (n_old, 3)).astype(np.float32); xyz_new = rng.normal(0, 1, (n_new, 3)).astype(np.float32)
    xyz_old[rng.random(n_old) < 0.2] = np.nan; xyz_new[rng.random(n_new) < 0.2] = np.nan
    oi, ni = PO.match_3d(old, new, xyz_old, xyz_new)
    best, d1, _, ps = PO.match_ratio(old, new)
    b32, d32, p8 = best.astype(np.int32), d1.astype(np.float32), ps.astype(np.uint8)
    a = np.zeros(n_new, np.int32); b = np.zeros(n_new, np.int32)
    m = lib.kth_match_3d(_p(b32), _p(d32), _p(p8), n_old, n_new, _p(xyz_old), _p(xyz_new), _p(a), _p(b))
    assert np.array_equal(a[:m], oi) and np.array_equal(b[:m], ni) and m > 20
    assert not np.isnan(xyz_old[oi]).any() and not np.isnan(xyz_new[ni]).any()
    # dropping the features without depth FIRST (the other order) gives a different match set: the order matters
    vo = ~np.isnan(xyz_old[:, 2]); vn = ~np.isnan(xyz_new[:, 2])
    bo, do_, _, po_ = PO.match_ratio(old[vo], new[vn])
    o2, n2 = PO.unique_matches(bo, do_, po_, int(vn.sum()))
    other = set(zip(np.flatnonzero(vo)[o2], np.flatnonzero(vn)[n2]))
    assert other != set(zip(oi, ni))


def test_project_inliers_truncates(lib):
    rows, cols = 20, 30
    dn = np.full((rows, cols), 1200, np.uint16); do = np.full((rows, cols), 2000, np.uint16); do[3, 7] = 0
    intr = np.array([50.0, 50.0, 15.0, 10.0], np.float32)
    kn = np.array([[4.9, 5.99], [10.2, 3.5], [1.0, 1.0]], np.float32); ko = np.array([[7.7, 3.2], [2.0, 2.0], [5.5, 5.5]], np.float32)
    inl = np.array([1, 1, 0], np.uint8)
    a = np.zeros((3, 3), np.float32); b = np.zeros((3, 3), np.float32)
    n = lib.kth_project_inliers(_p(kn), _p(ko), _p(inl), 3, _p(dn), _p(do), rows, cols, _p(intr), _p(a), _p(b))
    assert n == 1                          # the first pair's old pixel (7, 3) has no depth; the third is no inlier
    assert np.allclose(a[0], [1.2 * (10 - 15) / 50, 1.2 * (3 - 10) / 50, 1.2]) and np.allclose(b[0], [2.0 * (2 - 15) / 50, 2.0 * (2 - 10) / 50, 2.0])


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_pnp_equals_cv2(seed):
    import cv2
    rng = np.random.default_rng(seed)
    intr = np.array([264.0, 264.0, 160.0, 133.5]); n = 200
    R = Rotation.from_rotvec(rng.normal(0, 0.2, 3)).as_matrix(); t = rng.normal(0, 0.2, 3)
    uv = np.stack([rng.uniform(10, 310, n), rng.uniform(10, 230, n)], 1); z = rng.uniform(1.0, 4.0, n)
    p_old = np.stack([(uv[:, 0] - intr[2]) * z / intr[0], (uv[:, 1] - intr[3]) * z / intr[1], z], 1)
    p_new = (p_old - t) @ R
    uv = uv + rng.normal(0, 0.3, uv.shape)
    bad = rng.random(n) < 0.4
    p_new[bad] += rng.normal(0, 0.5, (bad.sum(), 3))
    Ro, to, inl = PO.pnp_ransac(p_new.astype(np.float32), p_old.astype(np.float32), uv.astype(np.float32), intr)
    K = np.array([[intr[0], 0, intr[2]], [0, intr[1], intr[3]], [0, 0, 1.0]])
    ok, rv, tv, inl2 = cv2.solvePnPRansac(p_new.astype(np.float32).astype(np.float64), uv.astype(np.float32).astype(np.float64), K, None,
                                          iterationsCount=500, reprojectionError=2.0)
    assert ok
    # both refine on the same inlier set: the same least-squares minimum
    ok, rv2, tv2 = cv2.solvePnP(p_new[inl].astype(np.float32).astype(np.float64), uv[inl].astype(np.float32).astype(np.float64), K, None,
                                rv, tv, useExtrinsicGuess=True, flags=cv2.SOLVEPNP_ITERATIVE)
    assert np.abs(cv2.Rodrigues(rv2)[0] - Ro).max() < 1e-6 and np.abs(tv2[:, 0] - to).max() < 1e-6
    # cv2 keeps the inliers of its best hypothesis; the device recomputes them after the refinement: they differ at the 2 px border only
    assert len(set(inl2[:, 0]) ^ set(np.flatnonzero(inl))) <= 0.02 * n


def test_fitness_equals_brute_force():
    from kintinuous_b200 import synth
    d0, _ = synth.render(0, 80, 60, noise=True); d1, _ = synth.render(4, 80, 60, noise=True)
    intr = synth.intrinsics(80, 60)
    T = np.eye(4); T[:3, 3] = [0.02, -0.01, 0.03]
    f, ns, nd = PO.fitness(d0, d1, intr, 0.04, T)
    S = PO.voxel_grid(PO.depth_cloud(d0, intr), 0.04) + T[:3, 3]; D = PO.voxel_grid(PO.depth_cloud(d1, intr), 0.04)
    assert (len(S), len(D)) == (ns, nd)
    assert abs(f - ((S[:, None, :] - D[None]) ** 2).sum(2).min(1).mean()) < 1e-12
