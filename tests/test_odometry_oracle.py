"""Pin the FP64 odometry reference (oracle/odometry_oracle.py) against what the reference's own CUDA operators computed
(tests/golden/rgbd_160x120.npz, ops_160x120.npz): the photometric correspondences, count and sigma, the photometric normal
equations within the oracle's per-entry bound, and the point-to-plane normal equations.  The GPU tests
(test_gpu_odometry_sums.py) then hold the product's kernels to the same oracle."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import odometry_oracle as oo


def _intensity(rgb):
    """rgb_to_intensity (kt_frontend.cuh): two fused multiply-adds in float, truncated.  The products of an 8-bit value and a float are
    exact in double, so each fma is one rounding to float here too."""
    c = rgb.astype(np.float64)
    f = lambda v: v.astype(np.float32).astype(np.float64)
    t = f(c[..., 2] * float(np.float32(0.299)))
    t = f(c[..., 0] * float(np.float32(0.114)) + t)
    t = f(c[..., 1] * float(np.float32(0.587)) + t)
    return t.astype(np.int64).astype(np.uint8)


@pytest.fixture(scope="module")
def rgbd():
    from kintinuous_b200 import synth
    g = np.load(os.path.join(GOLDEN, "rgbd_160x120.npz"))
    rows, cols = 120, 160
    rec = g["corres"]
    u0 = rec[:, 0:4].copy().view(np.int16).reshape(-1, 2)
    xy = rec[:, 4:8].copy().view(np.int16).reshape(-1, 2)
    diff = rec[:, 8:12].copy().view(np.float32).reshape(-1)
    valid = rec[:, 12] != 0
    _, c0 = synth.render(0, cols, rows)
    fx, fy, cx, cy = synth.intrinsics(cols, rows)
    return dict(g=g, rows=rows, cols=cols, u0=u0[:, 0].astype(np.int64), v0=u0[:, 1].astype(np.int64), xy=xy, diff=diff, valid=valid,
                last_image=_intensity(c0), kl=tuple(np.float32(v) for v in (fx, fy, cx, cy)),
                kd=tuple(float(np.float32(v)) for v in (fx, fy, cx, cy)))


def test_photometric_correspondences_match_the_reference(rgbd):
    """The correspondence test at the reference's warp (not the identity): same pixels, same last-frame pixel, same diff, except
    where the oracle flags a rounding or threshold tie; count and sigma exactly the reference's when there is none."""
    r, g = rgbd, rgbd["g"]
    rows, cols = r["rows"], r["cols"]
    last_depth = g["cloud"][..., 2]
    assert (r["last_image"] != 0).mean() > 0.9
    corr = oo.photometric_correspondences(g["intensity"], g["depth_f"], g["dIdx"], g["dIdy"], last_depth, r["last_image"], 2, g["krk"], g["kt"])
    valid = corr["valid"].reshape(-1); amb = corr["ambiguous"].reshape(-1)
    assert int(amb.sum()) <= 20, int(amb.sum())              # ties within the float error of an edge: a few in 19 200
    sure = ~amb
    assert (valid[sure] == r["valid"][sure]).all(), int((valid[sure] != r["valid"][sure]).sum())
    v = valid & sure
    assert (corr["u0"].reshape(-1)[v] == r["u0"][v]).all() and (corr["v0"].reshape(-1)[v] == r["v0"][v]).all()
    assert (corr["diff"].reshape(-1)[v] == r["diff"][v]).all()
    yy, xx = np.divmod(np.arange(rows * cols), cols)
    assert (r["xy"][r["valid"], 0] == xx[r["valid"]]).all() and (r["xy"][r["valid"], 1] == yy[r["valid"]]).all()
    count, sigma, n_amb = oo.count_and_sigma(corr)
    if n_amb == 0:
        assert (sigma, count) == tuple(int(x) for x in g["sigma_count"])


def _reference_correspondences(r):
    rows, cols = r["rows"], r["cols"]
    return dict(valid=r["valid"].reshape(rows, cols), ambiguous=np.zeros((rows, cols), bool), u0=r["u0"].reshape(rows, cols),
                v0=r["v0"].reshape(rows, cols), diff=r["diff"].astype(np.float64).reshape(rows, cols),
                gx=r["g"]["dIdx"].astype(np.int64), gy=r["g"]["dIdy"].astype(np.int64))


def test_photometric_normal_equations_within_the_bound(rgbd):
    """FP64 rows and sums from the reference's own correspondences and point cloud: the reference's float A / b lie within the
    oracle's bound, and the bound is tight (a wrong weight, gradient scale or point would be far outside it)."""
    r, g = rgbd, rgbd["g"]
    corr = _reference_correspondences(r)
    count, sigma_sq, _ = oo.count_and_sigma(corr)
    assert (sigma_sq, count) == tuple(int(x) for x in g["sigma_count"])
    sigma = oo.q3_sigma(count, sigma_sq)
    assert sigma == np.float32(np.sqrt(count))
    s = oo.photometric_system(corr, sigma, None, r["kl"], r["kd"], cloud=g["cloud"])
    for mine, bound, ref in ((s.A, s.dA, g["rgb_A"]), (s.b, s.db, g["rgb_b"])):
        err = np.abs(ref.astype(np.float64) - mine)
        assert (err <= bound).all(), float((err / bound).max())
    # the reference's float tree lies well inside: the bound is a few ulps of S_ij, not a loose multiple of |A|
    assert (s.dA <= 1e-4 * np.abs(s.A).max()).all()
    # the rows themselves are pinned: the weight without sigma (the Q3 regime of a repeated frame) moves A by far more than the bound
    s1 = oo.photometric_system(corr, 1.0, None, r["kl"], r["kd"], cloud=g["cloud"])
    assert (np.abs(s1.A - g["rgb_A"]) > s.dA).any()


def test_photometric_rows_from_depth_equal_rows_from_the_cloud(rgbd):
    """The whole-frame kernel rebuilds the last-frame point from its depth with projectToPointCloud's arithmetic instead of reading the
    cloud: the oracle's two forms agree to the bound."""
    r, g = rgbd, rgbd["g"]
    corr = _reference_correspondences(r)
    count, sigma_sq, _ = oo.count_and_sigma(corr)
    sigma = oo.q3_sigma(count, sigma_sq)
    a = oo.photometric_system(corr, sigma, None, r["kl"], r["kd"], cloud=g["cloud"])
    b = oo.photometric_system(corr, sigma, g["cloud"][..., 2], r["kl"], r["kd"])
    assert (np.abs(a.P - b.P) <= a.bound).all()


def test_q3_sigma_rule():
    assert oo.q3_sigma(1000, 0) == 1.0                       # every diff zero: weight 1 / (1 + |diff|)
    assert oo.q3_sigma(1000, 5) == np.float32(np.sqrt(1000.0))
    assert oo.q3_sigma(1000, -7) == np.float32(np.sqrt(1000.0))   # a wrapped sum is still not zero
    assert oo.q3_sigma(0, 0) == 0.0


def test_identity_warp_maps_a_pixel_to_itself():
    from kintinuous_b200 import synth
    for level in range(4):
        kl, kd = oo.level_intrinsics(*synth.intrinsics(640, 480), level)
        krk, kt = oo.build_warp(np.eye(4), *kd)
        rows, cols = 480 >> level, 640 >> level
        img = np.full((rows, cols), 100, np.uint8)
        depth = np.full((rows, cols), 1.5, np.float32)
        grad = np.full((rows, cols), 2000, np.int16)
        corr = oo.photometric_correspondences(img, depth, grad, grad, depth, img, level, krk, kt)
        y, x = np.mgrid[0:rows, 0:cols]
        v = corr["valid"]
        assert not corr["ambiguous"].any() and v.sum() == (rows - 1) * (cols - 5)      # x < cols - 5, y < rows - 1 (reduce.cu:711)
        assert (corr["u0"][v] == x[v]).all() and (corr["v0"][v] == y[v]).all()


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _f(a):
    return np.ascontiguousarray(np.asarray(a, np.float32).reshape(-1))


def test_icp_normal_equations_vs_reference(cpu_oracle):
    """The inputs of test_oracle_golden.py::test_icp_normal_equations (maps rebuilt with the C++ oracle from the golden filtered depth),
    and the same tolerance against the reference's float reduction."""
    from kintinuous_b200 import synth
    G = np.load(os.path.join(GOLDEN, "ops_160x120.npz"))
    rows, cols = 120, 160
    lib = cpu_oracle.lib
    intr = np.array(synth.intrinsics(cols, rows), np.float32)
    R0 = np.eye(3, dtype=np.float32); t0 = np.array([3, 3, 3], np.float32)
    vm = np.ascontiguousarray(G["vmap"]); nm = np.ascontiguousarray(G["nmap"])
    mv = np.zeros_like(vm); mn = np.zeros_like(vm)
    lib.ktoracle_transform_maps(_p(vm), _p(nm), _p(_f(R0)), _p(_f(t0)), _p(mv), _p(mn), rows, cols)
    d3, _ = synth.render(12, cols, rows)
    f3 = np.zeros((rows, cols), np.uint16); lib.ktoracle_bilateral(_p(d3), _p(f3), rows, cols)
    cv = np.zeros_like(vm); cn = np.zeros_like(vm)
    lib.ktoracle_vmap(_p(f3), _p(cv), rows, cols, _p(intr)); lib.ktoracle_nmap(_p(cv), _p(cn), rows, cols)
    s = oo.icp_system(cv.reshape(3, rows, cols), cn.reshape(3, rows, cols), mv.reshape(3, rows, cols), mn.reshape(3, rows, cols), R0, t0, intr)
    gA, gb, gres = G["icp_A"].astype(np.float64), G["icp_b"].astype(np.float64), G["icp_res"]
    assert abs(s.count - gres[1]) <= 0.002 * gres[1] + s.extra["ambiguous"]
    assert np.abs(s.A - gA).max() <= 2e-3 * np.abs(gA).max()
    assert np.abs(s.b - gb).max() <= 2e-3 * np.abs(gb).max() + 1e-3
    assert abs(s.residual - gres[0]) <= 2e-3 * abs(gres[0]) + 1e-6


def test_merge_and_pose_propagation():
    """The -ri merge weights (100 on A, 10 on b) and the pose after one step: an exactly solvable system gives its increment back."""
    rng = np.random.default_rng(3)
    J = rng.standard_normal((200, 6)); r = rng.standard_normal(200) * 1e-3
    def system(J, r):
        P, _, _ = oo._products(np.concatenate([J, r[:, None]], 1), np.zeros((len(r), 7)))
        return oo.System(P, np.full(29, 1e-9), len(r))
    a, b = system(J, r), system(J * 0.5, r * 2)
    m = oo.merge(a, b)
    assert np.allclose(m.A, a.A + 100 * b.A) and np.allclose(m.b, a.b + 10 * b.b)
    Rp = np.eye(3); tp = np.array([3.0, 3.0, 3.0])
    Rc, tc, tol_R, tol_t, x = oo.pose_after_one_iteration(a, Rp, tp)
    assert np.allclose(x, np.linalg.lstsq(J, r, rcond=None)[0], atol=1e-12)
    assert 0 < tol_t < 1e-5 and 0 < tol_R < 1e-5
    Rc0, tc0, _, _, x0 = oo.pose_after_one_iteration(oo.System(np.zeros(29), np.zeros(29), 0), Rp, tp)
    assert (x0 == 0).all() and (Rc0 == Rp).all() and (tc0 == tp).all()
