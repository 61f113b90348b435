"""tests/slice_knn_reference.py (the exact reference tests/test_gpu_slice_knn.py holds kt_slice.cu to) pinned on the CPU: its k-NN
against brute force, ties included; its eigen33 against numpy.linalg.eigh; its leaf grid, centroids, colours and neighbour sets against
oracle/kt_slice_oracle.cpp wherever that oracle is exact; and every GPU scene reaching the search path it was built for."""
import os
import sys

import numpy as np
import pytest

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tests"))
import slice_knn_reference as R  # noqa: E402
from slice_cloud import make_cloud  # noqa: E402
from test_gpu_slice_knn import SCENES, TRACKER_LEAF, margin_sliver  # noqa: E402


def _brute(xyz, k):
    n = len(xyz)
    q = np.repeat(np.arange(n), n).reshape(n, n); nb = np.tile(np.arange(n), n).reshape(n, n)
    packed = np.sort(R._pack(R.keys32(xyz, q, nb), nb), axis=1)[:, :k]
    return (packed & np.uint64(0xffffffff)).astype(np.int64), (packed >> np.uint64(32)).astype(np.uint32).view(np.float32)


@pytest.mark.parametrize("case", ["random", "far", "lattice", "duplicates"])
def test_knn_is_brute_force(case):
    rng = np.random.default_rng(3)
    for n, k in ((5, 20), (40, 20), (300, 20), (300, 33), (300, 1)):
        if case == "random":
            xyz = rng.uniform(-1, 1, (n, 3))
        elif case == "far":
            xyz = rng.uniform(-1, 1, (n, 3)) * 0.05 + 1600.0
        elif case == "lattice":                                   # exact float distances: ties everywhere, decided by the slot
            xyz = rng.permutation(np.stack(np.meshgrid(*[np.arange(8)] * 3, indexing="ij"), -1).reshape(-1, 3))[:n] * 0.25
        else:                                                     # coincident points: key 0 for several slots
            xyz = rng.uniform(-1, 1, (n, 3))[rng.integers(0, max(1, n // 3), n)]
        xyz = xyz.astype(np.float32)
        s, d = R.knn(xyz, k)
        bs, bd = _brute(xyz, min(k, n))
        assert np.array_equal(s, bs) and np.array_equal(d.view(np.uint32), bd.view(np.uint32)), (case, n, k)
        if case == "lattice" and (n, k) == (300, 20):
            assert (d[:, -1] == _brute(xyz, k + 1)[1][:, -1]).sum() > 100        # the k-th distance is tied with the (k+1)-th often


def test_eigen33_matches_eigh():
    rng = np.random.default_rng(11)
    mats = []
    for _ in range(500):
        w = np.sort(rng.uniform(0.01, 1.0, 3)) * 10.0 ** rng.uniform(-8, 2)
        w[1] = max(w[1], w[0] + 0.05 * w[2]); w[2] = max(w[2], w[1] * 1.05)
        q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        mats.append((q * w) @ q.T)
    mats = np.array(mats)
    ev, v = R.eigen33_smallest(mats.reshape(-1, 9))
    w, u = np.linalg.eigh(mats)
    assert np.allclose(np.linalg.norm(v, axis=1), 1.0, atol=1e-14)
    assert (np.abs(ev - w[:, 0]) <= 1e-12 * w[:, 2]).all()
    ang = np.arctan2(np.linalg.norm(np.cross(v, u[:, :, 0]), axis=1), np.abs((v * u[:, :, 0]).sum(1)))
    assert ang.max() < 1e-10, ang.max()
    # a planar neighbourhood: computeRoots2, lambda0 = 0 and the normal of the plane
    p = np.stack([rng.normal(size=20), rng.normal(size=20), np.zeros(20)])
    ev, v = R.eigen33_smallest(np.cov(p, bias=True).reshape(1, 9))
    assert ev[0] == 0.0 and abs(abs(v[0, 2]) - 1.0) < 1e-15


@pytest.fixture(scope="module")
def oracle():
    from oracle import refbind
    import subprocess
    if not os.path.exists(os.path.join(ROOT, "oracle", "libkt_slice_oracle.so")):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "libkt_slice_oracle.so"])
    return refbind.SliceOracle(), refbind


@pytest.mark.parametrize("offset", [(1.7, -0.9, 2.3), (800.0, -800.0, 1600.0)])
def test_grid_and_neighbours_match_the_oracle(oracle, offset):
    o, rb = oracle
    pts = make_cloud(n_side=100, offset=offset, point_dtype=rb.POINT_DTYPE)
    ref = R.leaf_grid(pts, 8, TRACKER_LEAF)
    vg, min_b, div_b = o.voxel_grid(o.weight_cull(pts, 8), TRACKER_LEAF)
    assert len(vg) == len(ref["xyz"]) and (min_b == ref["min_b"]).all() and (div_b == ref["div_b"]).all()
    oxyz = np.stack([vg["x"], vg["y"], vg["z"]], -1)
    # the oracle sums floats: exact for a leaf of one point, within float rounding of the mean otherwise
    one = ref["count"] == 1
    assert one.sum() > 100 and np.array_equal(oxyz[one].view(np.uint32), ref["xyz"][one].view(np.uint32))
    assert np.abs(oxyz.astype(np.float64) - ref["xyz"]).max() <= 4 * np.spacing(np.abs(ref["xyz"]).max())
    for c, ch in enumerate("rgb"):
        assert np.array_equal(vg[ch], ref["rgb"][:, c]), ch                       # integer sums below 2^24: exact in both
    # neighbour sets over the oracle's own centroids: the oracle's PCL-float normal of a point over the whole cloud is bit for bit its
    # normal over just the reference's neighbours (kept in slot order, so the oracle ranks and sums them in the same order) iff the sets agree
    slots, _ = R.knn(oxyz, 20)
    full = o.normals(vg, 20, TRACKER_LEAF)
    sample = np.random.default_rng(2).choice(len(vg), 400, replace=False)
    for i in sample:
        sub = np.sort(slots[i])
        one_n = o.normals(vg[sub], 20, TRACKER_LEAF)[int(np.flatnonzero(sub == i)[0])]
        for f in ("nx", "ny", "nz", "curvature"):
            assert one_n[f].view(np.uint32) == full[i][f].view(np.uint32), (i, f)


@pytest.mark.parametrize("scene", list(SCENES))
def test_scene_takes_its_search_paths(oracle, scene):
    """Each GPU scene sends well-conditioned points down the path it was built for, and wherever the kernel's stop rule (with its
    0.001-leaf margin) stops, its cube already holds the exact neighbours."""
    _, rb = oracle
    build, cull, leaf, k, expect, _ = SCENES[scene]
    ref = R.process_slice(build(rb.POINT_DTYPE), cull, leaf, k)
    assert not ref["stop_unsafe"].any() and not ref["stop_wrong"].any(), (scene, int(ref["stop_unsafe"].sum()), int(ref["stop_wrong"].sum()))
    missing, _ = R.unmet(ref, expect, 1e-3)
    assert not missing, (scene, missing)


def test_margin_sliver_defeats_a_fixed_margin(oracle):
    """With the fixed 0.001-leaf margin the stop rule once had, the sliver scene stops on a cube that misses an exact neighbour in every
    copy (the premise check sees it); the margin derived from the grid's extent (0.001 + 4 ulp(max |x * inv_leaf|)) stops one radius later."""
    _, rb = oracle
    pts = margin_sliver(rb.POINT_DTYPE)
    old = R.process_slice(pts, 8, 0.01, 3, margin=0.001)
    assert old["stop_unsafe"].sum() == old["stop_wrong"].sum() == 4
    assert (old["stop_slack"][old["stop_unsafe"]] < -0.001).all()
    new = R.process_slice(pts, 8, 0.01, 3)
    assert new["margin"] == np.float32(0.001) + np.float32(4 * 2.0 ** -7)
    assert not new["stop_unsafe"].any() and not new["stop_wrong"].any()
    # what a kernel with the fixed margin would return: the 3 nearest inside the +-5 cube, whose normal is far from the exact one
    for q in np.flatnonzero(old["stop_unsafe"]):
        assert R.PATHS[old["path"][q]] == "stop5"
        cube = np.flatnonzero((np.abs(old["ijk"] - old["ijk"][q]) <= 5).all(1))
        picked = cube[np.lexsort((cube, R.keys32(old["xyz"], np.full(len(cube), q), cube)))[:3]]
        nrm, _, _ = R.normals(old["xyz"][np.r_[q, picked]], np.arange(1, 4)[None, :].repeat(4, 0))
        assert abs(float(nrm[0] @ new["normal"][q])) < 0.1                              # ~90 degrees apart

def test_fallback_paths_are_all_covered():
    assert {"covers", "overflow", "rcap", "isolated"} <= {p for e in SCENES.values() for p in e[4]}
