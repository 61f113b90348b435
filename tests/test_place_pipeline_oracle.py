"""The oracle's additions for loop detection's stages (oracle/place_oracle.py), without a GPU: SURF's decision margins, the device's
keypoints_3d, project_inliers against kt_place.hpp, and verify -- the whole of place_process after retrieval -- on a rendered pair with a
known relative pose."""
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
    lib.kth_lookup_3d.argtypes = [C.c_float, C.c_float, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _blob_image(n=160, centres=((60.3, 80.0),), sigma=4.0):
    y, x = np.mgrid[0:n, 0:n].astype(np.float64)
    img = np.full((n, n), 230.0)
    for cx, cy in centres:
        img -= 200.0 * np.exp(-((x - cx) ** 2 + (y - cy) ** 2) / (2 * sigma ** 2))
    return np.repeat(np.rint(img)[..., None], 3, -1).astype(np.uint8)


def test_orientation_margin_is_zero_exactly_at_a_tie():
    # an image symmetric under column x <-> 159 - x: at x = 80 the Haar responses of mirrored samples are (-dx, dy), so the windows at
    # 5k and 180 - 5k degrees have mirrored members and the same squared length -- an exact tie between windows with other members
    rng = np.random.default_rng(2)
    g = np.kron(rng.integers(20, 235, (40, 20)), np.ones((4, 4))).astype(np.uint8)
    g = np.concatenate([g, g[:, ::-1]], 1)
    I = PO.integral(PO.grey(np.repeat(g[..., None], 3, -1)))
    ties = 0
    for y in np.arange(60.0, 100.0, 2.3):
        th, _, m = PO.describe(I, 80.0, y, 20.0, 160, 160, margins=True)
        vertical = abs(abs(th) - np.pi / 2) < 1e-12                 # the best window is its own mirror image: no twin
        assert (m["ori"] == 0.0) != vertical, (y, th, m)
        ties += not vertical
    assert ties >= 5
    # off the axis of symmetry there is no tie
    _, _, m = PO.describe(I, 77.3, 80.3, 20.0, 160, 160, margins=True)
    assert m["ori"] > 1e-6, m


def test_sample_margin_is_zero_exactly_on_a_rounding_boundary():
    I = PO.integral(PO.grey(_blob_image()))
    _, _, m = PO.describe(I, 60.5, 80.0, 18.0, 160, 160, margins=True)         # sample (0, 0) of the orientation disc lies on x = 60.5
    assert m["sample"] == 0.0 and m["sample_slack"] < 0, m
    _, _, m = PO.describe(I, 60.3, 80.0, 18.0, 160, 160, margins=True)
    assert m["sample"] > 0.0, m


def test_surf_margins_leave_the_outputs_alone():
    from kintinuous_b200 import synth
    _, rgb = synth.render_at(*synth.pose(3), 160, 120, noise=True, texture=synth.cell_texture)
    kp, desc = PO.surf(rgb, 100)
    kp2, desc2, mg = PO.surf(rgb, 100, margins=True)
    assert np.array_equal(kp, kp2) and np.array_equal(desc, desc2) and len(kp) > 10
    assert set(mg) == {"ori", "ori_bound", "ori_edge", "sample", "sample_slack", "sample_turn"}
    assert all(len(v) == len(kp) for v in mg.values())
    assert (mg["ori"] >= 0).all() and (mg["ori"] <= 1).all() and (mg["sample"] >= 0).all() and (mg["sample"] <= 0.5).all()


def test_keypoints_3d_equals_lookup_and_the_header(lib):
    rows, cols = 10, 12
    depth = np.zeros((rows, cols), np.uint16); depth[4, 5] = 1500; depth[4, 6] = 10000; depth[4, 7] = 9999; depth[3, 3] = 65535
    depth[0, 0] = 800; depth[rows - 1, cols - 1] = 2345; depth[5, 5] = 0
    intr = np.array([100.0, 101.5, 6.0, 5.0], np.float32)
    h = np.float32(0.5); e = np.float32(1e-6)
    xs = []
    for u, v in ((5, 4), (6, 4), (7, 4), (3, 3), (0, 0), (cols - 1, rows - 1), (5, 5)):
        for dx in (-h, h, np.nextafter(-h, np.float32(0)), np.nextafter(h, np.float32(0)), np.float32(0), -e, e):
            xs.append((np.float32(u) + dx, np.float32(v)))
            xs.append((np.float32(u), np.float32(v) + dx))
    xs += [(-0.4, 0.0), (-0.5, 0.0), (cols - 0.5, rows - 1.0), (cols - 0.6, rows - 1.0), (0.0, -0.49)]
    kp = np.zeros((len(xs), 6), np.float32); kp[:, :2] = np.array(xs, np.float32)
    got = PO.keypoints_3d(kp, depth, intr)
    assert got.dtype == np.float32 and got.shape == (len(xs), 3)
    n_point = 0
    for i, (x, y) in enumerate(kp[:, :2]):
        o = PO.lookup_3d(x, y, depth, intr)
        out = np.zeros(3, np.float32)
        ok = lib.kth_lookup_3d(float(x), float(y), _p(depth), rows, cols, _p(intr), _p(out))
        assert bool(ok) == (o is not None) == (not np.isnan(got[i]).any()), (x, y)
        if ok:
            n_point += 1
            assert np.array_equal(got[i], o) and np.array_equal(got[i], out), (x, y, got[i], o, out)
        else:
            assert np.isnan(got[i]).all()
    # depth 0, z = 10 m and z > 10 m have no point; the strict half pixel none; what is left has one
    assert 10 < n_point < len(xs) - 20


def test_project_inliers_equals_the_header(lib):
    rng = np.random.default_rng(4)
    rows, cols, n = 30, 40, 300
    dn = rng.integers(0, 4000, (rows, cols)).astype(np.uint16); do = rng.integers(0, 4000, (rows, cols)).astype(np.uint16)
    dn[rng.random((rows, cols)) < 0.2] = 0; do[rng.random((rows, cols)) < 0.2] = 0
    intr = np.array([35.0, 36.0, 19.5, 14.5], np.float32)
    kn = np.stack([rng.uniform(-1.5, cols + 0.5, n), rng.uniform(-1.5, rows + 0.5, n)], 1).astype(np.float32)
    ko = np.stack([rng.uniform(-1.5, cols + 0.5, n), rng.uniform(-1.5, rows + 0.5, n)], 1).astype(np.float32)
    kn[:20] = np.floor(kn[:20]) + np.float32(0.999999); ko[20:40] = np.float32(-0.7)                    # truncation, not rounding
    inl = (rng.random(n) < 0.7).astype(np.uint8)
    a = np.zeros((n, 3), np.float32); b = np.zeros((n, 3), np.float32)
    m = lib.kth_project_inliers(_p(kn), _p(ko), _p(inl), n, _p(dn), _p(do), rows, cols, _p(intr), _p(a), _p(b))
    ea, eb = PO.project_inliers(kn, ko, inl, dn, do, intr)
    assert m == len(ea) > 50
    assert np.array_equal(a[:m], ea) and np.array_equal(b[:m], eb)


def _cpu_maps(lib, depth, intr, levels=4):
    """The reference's front end on the CPU (bilateral, pyrDown, createVMap, createNMap): per level (vmap, nmap) [3, rows, cols]."""
    rows, cols = depth.shape
    d = np.zeros((rows, cols), np.uint16); lib.ktoracle_bilateral(_p(np.ascontiguousarray(depth)), _p(d), rows, cols)
    out = []
    for l in range(levels):
        r, c = rows >> l, cols >> l
        if l:
            nd = np.zeros((r, c), np.uint16); lib.ktoracle_pyrdown(_p(d), _p(nd), r * 2, c * 2); d = nd
        k = np.array([intr[0] / (1 << l), intr[1] / (1 << l), intr[2] / (1 << l), intr[3] / (1 << l)], np.float32)
        vm = np.zeros((3 * r, c), np.float32); nm = np.zeros_like(vm)
        lib.ktoracle_vmap(_p(d), _p(vm), r, c, _p(k)); lib.ktoracle_nmap(_p(vm), _p(nm), r, c)
        out.append((vm.reshape(3, r, c), nm.reshape(3, r, c)))
    return out


def test_verify_recovers_a_rendered_relative_pose(cpu_oracle):
    from kintinuous_b200 import synth
    cols, rows = 320, 240
    intr = np.array(synth.intrinsics(cols, rows), np.float32)
    R1 = Rotation.from_rotvec([0.0, np.deg2rad(4.0), 0.0]).as_matrix(); t1 = np.array([0.05, 0.0, 0.02])
    d_old, c_old = synth.render_at(np.eye(3), np.zeros(3), cols, rows, noise=True, noise_seed=1, texture=synth.cell_texture)
    d_new, c_new = synth.render_at(R1, t1, cols, rows, noise=True, noise_seed=2, texture=synth.cell_texture)
    ko, do_ = PO.surf(c_old, 1000); kn, dn = PO.surf(c_new, 1000)
    mo, mn = _cpu_maps(cpu_oracle.lib, d_old, intr), _cpu_maps(cpu_oracle.lib, d_new, intr)
    v = PO.verify(d_old, ko, do_, d_new, kn, dn, intr, mo, mn, voxel=6.0 / 256)
    assert v["stage"] == "loop", {k: v[k] for k in ("stage", "matches") if k in v}
    assert v["margin_matches"] > 0 and v["margin_ratio"] > 0 and v["margin_fitness"] > 0
    # C: the old camera in the new one, inv(P_new) P_old with P_old = I
    P1 = np.eye(4); P1[:3, :3] = R1; P1[:3, 3] = t1
    gt = np.linalg.inv(P1)
    C_ = v["C"]
    assert np.linalg.norm(C_[:3, 3] - gt[:3, 3]) < 5e-3, (C_, gt)
    assert np.linalg.norm(Rotation.from_matrix(C_[:3, :3].T @ gt[:3, :3]).as_rotvec()) < np.deg2rad(0.3)
    # the dense check improves on PnP alone
    Tp = np.eye(4); Tp[:3, :3] = v["R_pnp"]; Tp[:3, 3] = v["t_pnp"]
    assert np.linalg.norm(C_[:3, 3] - gt[:3, 3]) <= np.linalg.norm(np.linalg.inv(Tp)[:3, 3] - gt[:3, 3]) + 1e-3
    # the inliers back-project to the same world points within the depth noise
    a, b = v["inliers1"], v["inliers2"]
    assert len(a) > 20 and len(a) == len(b)
    moved = b @ C_[:3, :3].T + C_[:3, 3]
    assert np.median(np.linalg.norm(moved - a, axis=1)) < 0.03
    # a pair that does not overlap stops at the match count
    d_far, c_far = synth.render_at(Rotation.from_rotvec([0.0, np.pi, 0.0]).as_matrix(), np.zeros(3), cols, rows, noise=True, texture=synth.cell_texture)
    kf, df = PO.surf(c_far, 1000)
    w = PO.verify(d_old, ko, do_, d_far, kf, df, intr, mo, _cpu_maps(cpu_oracle.lib, d_far, intr), voxel=6.0 / 256)
    assert w["stage"] in ("matches", "inliers", "fitness") and w["stage"] != "loop"
