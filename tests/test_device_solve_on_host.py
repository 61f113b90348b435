"""The Gauss-Newton step that runs INSIDE the odometry kernels (kintinuous_b200/csrc/kt_solve.cuh: 6x6 LDL^T in FP64, Rodrigues,
pose composition) replaces host arithmetic the reference gets from Eigen and OpenCV (ICPOdometry.cpp:127-178, OdometryProvider.h:54-68).
Its source compiles for the host as well (tests/cpp/solve_host.cu), so it is checked here on the CPU against numpy, cv2 and the
pinned oracle restatements -- including the cases Eigen's pivoted LDLT treats specially (rank-deficient normal matrices)."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import ROOT


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def solve_lib():
    out = os.path.join(ROOT, "tests", "cpp", "_build")
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, "libkt_solve_host.so")
    src = os.path.join(ROOT, "tests", "cpp", "solve_host.cu")
    hdr = os.path.join(ROOT, "kintinuous_b200", "csrc", "kt_solve.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"          # the Makefile's default too
        subprocess.check_call([nvcc, "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "kintinuous_b200", "csrc"),
                               "-gencode", "arch=compute_90a,code=sm_90a", "-o", so, src])
    return C.CDLL(so)


def _normal_matrix(rng, scale=1.0, rank=6):
    J = rng.standard_normal((300, 6)) * np.array([1, 1, 1, 0.3, 0.3, 0.3])
    if rank < 6:
        J[:, rank:] = 0.0
    return scale * (J.T @ J)


def test_ldlt6_matches_numpy_and_the_oracle(solve_lib, cpu_oracle):
    rng = np.random.default_rng(20260922)
    for trial in range(100):
        A = _normal_matrix(rng, 1e4 if trial % 5 == 0 else 1.0)
        b = rng.standard_normal(6) * (100.0 if trial % 3 == 0 else 1.0)
        x = np.zeros(6); xo = np.zeros(6)
        solve_lib.kts_ldlt6_solve(_p(np.ascontiguousarray(A)), _p(b), _p(x))
        cpu_oracle.lib.ktoracle_ldlt6_solve(_p(np.ascontiguousarray(A)), _p(b), _p(xo))
        ref = np.linalg.solve(A, b)
        assert np.allclose(x, ref, rtol=1e-9, atol=1e-12)
        # unpivoted (device) vs diagonally pivoted (Eigen restatement): far below the float the pose is rounded to
        assert np.abs(x - xo).max() <= 1e-10 * max(1.0, np.abs(xo).max())


def test_ldlt6_degenerate_systems_behave_like_eigen(solve_lib, cpu_oracle):
    """No inliers (A = 0, b = 0): zero increment.  Rank-deficient A with a consistent b: both give a solution of the system."""
    x = np.ones(6)
    solve_lib.kts_ldlt6_solve(_p(np.zeros((6, 6))), _p(np.zeros(6)), _p(x))
    assert (x == 0).all()
    rng = np.random.default_rng(3)
    for rank in (3, 5):
        A = _normal_matrix(rng, rank=rank)
        xt = np.zeros(6); xt[:rank] = rng.standard_normal(rank)
        b = A @ xt
        x = np.zeros(6); xo = np.zeros(6)
        solve_lib.kts_ldlt6_solve(_p(np.ascontiguousarray(A)), _p(b), _p(x))
        cpu_oracle.lib.ktoracle_ldlt6_solve(_p(np.ascontiguousarray(A)), _p(b), _p(xo))
        assert np.isfinite(x).all()
        assert np.allclose(A @ x, b, rtol=1e-8, atol=1e-8) and np.allclose(A @ xo, b, rtol=1e-8, atol=1e-8)
        assert np.allclose(x, xo, atol=1e-8)


def test_rodrigues_matches_cv2(solve_lib, cpu_oracle):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(1)
    for scale in (0.0, 1e-17, 1e-12, 1e-6, 1e-3, 0.1, 1.0, 3.0):
        for _ in range(10):
            r = rng.standard_normal(3) * scale
            R = np.zeros(9); Ro = np.zeros(9)
            solve_lib.kts_rodrigues(_p(r), _p(R))
            cpu_oracle.lib.ktoracle_rodrigues(_p(r), _p(Ro))
            Rcv, _ = cv2.Rodrigues(r.reshape(3, 1))
            assert np.abs(R.reshape(3, 3) - Rcv).max() < 1e-14
            assert np.abs(R - Ro).max() < 1e-15


def test_mat3f_inverse_is_bit_identical_to_the_eigen_restatement(solve_lib, cpu_oracle):
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(2)
    for _ in range(200):
        m = Rotation.from_rotvec(rng.standard_normal(3) * rng.choice([1e-3, 0.1, 2.0])).as_matrix().astype(np.float32)
        a = np.zeros(9, np.float32); b = np.zeros(9, np.float32)
        solve_lib.kts_mat3f_inverse(_p(np.ascontiguousarray(m)), _p(a))
        cpu_oracle.lib.ktoracle_mat3_inverse(_p(np.ascontiguousarray(m)), _p(b))
        assert (a.view(np.uint32) == b.view(np.uint32)).all()


def test_unpack_order(solve_lib):
    s = np.arange(27, dtype=np.float32) + 1
    A = np.zeros(36, np.float32); b = np.zeros(6, np.float32)
    solve_lib.kts_unpack(_p(s), _p(A), _p(b))
    A = A.reshape(6, 6)
    assert (A == A.T).all()
    k = 0
    for i in range(6):                                  # internal.h:101-106 order: aa ab ac ad ae af ag bb ...
        for j in range(i, 7):
            assert (b[i] if j == 6 else A[i, j]) == s[k]
            k += 1


def test_pose_update_follows_the_reference_formulas(solve_lib):
    """resultRt <- [Rodrigues(x[3:]) | x[:3]] * resultRt (double); [Rcurr | tcurr] = [Rprev | tprev] * inverse(resultRt) (float)."""
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(5)
    for _ in range(50):
        A = _normal_matrix(rng)
        xt = rng.standard_normal(6) * np.array([0.02, 0.02, 0.02, 0.01, 0.01, 0.01])
        b = A @ xt
        Rt = np.eye(4)
        Rt[:3, :3] = Rotation.from_rotvec(rng.standard_normal(3) * 0.02).as_matrix(); Rt[:3, 3] = rng.standard_normal(3) * 0.01
        Rprev = Rotation.from_rotvec(rng.standard_normal(3)).as_matrix().astype(np.float32)
        tprev = (rng.standard_normal(3) + 3).astype(np.float32)
        res = Rt.copy().reshape(-1)
        Rc = np.zeros(9, np.float32); tc = np.zeros(3, np.float32)
        solve_lib.kts_update(_p(np.ascontiguousarray(A)), _p(b), _p(res), _p(np.ascontiguousarray(Rprev)), _p(tprev), _p(Rc), _p(tc))
        cur = np.eye(4); cur[:3, :3] = Rotation.from_rotvec(xt[3:]).as_matrix(); cur[:3, 3] = xt[:3]
        want = cur @ Rt
        assert np.abs(res.reshape(4, 4) - want).max() < 1e-9
        inv = np.linalg.inv(want)
        assert np.abs(Rc.reshape(3, 3) - Rprev.astype(np.float64) @ inv[:3, :3]).max() < 1e-6
        assert np.abs(tc - (Rprev.astype(np.float64) @ inv[:3, 3] + tprev)).max() < 1e-6


def test_trimmed_forms_agree_with_the_closed_forms(solve_lib):
    """The whole-frame kernels run the latency-trimmed step (kt_solve.cuh: gauss_newton_update_fast): series Rodrigues below 0.5 rad
    (closed form above), three-row product.  Against cv2.Rodrigues: 2 ulp of the matrix entries; against the plain step: the float pose
    may differ in its last bit only where the double intermediate sits on a rounding boundary."""
    cv2 = pytest.importorskip("cv2")
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(9)
    for scale in (0.0, 1e-17, 1e-9, 1e-4, 1e-2, 0.1, 0.28, 0.29, 0.5, 1.0, 3.0):       # 0.28 / 0.29: either side of |r|^2 = 0.25 for unit-ish directions
        for _ in range(20):
            r = rng.standard_normal(3); r = r / np.linalg.norm(r) * scale * (1.0 + 0.5 * rng.random())
            R = np.zeros(9)
            solve_lib.kts_rodrigues_fast(_p(r), _p(R))
            Rcv, _ = cv2.Rodrigues(r.reshape(3, 1))
            assert np.abs(R.reshape(3, 3) - Rcv).max() < 5e-16, (scale, np.abs(R.reshape(3, 3) - Rcv).max())
    worst = 0.0
    for _ in range(200):
        A = _normal_matrix(rng, rng.choice([1.0, 1e3, 1e5]))
        xt = rng.standard_normal(6) * np.array([0.02, 0.02, 0.02, 0.01, 0.01, 0.01]) * rng.choice([1.0, 1e-3])
        b = A @ xt
        Rt = np.eye(4)
        Rt[:3, :3] = Rotation.from_rotvec(rng.standard_normal(3) * 0.02).as_matrix(); Rt[:3, 3] = rng.standard_normal(3) * 0.01
        Rprev = Rotation.from_rotvec(rng.standard_normal(3)).as_matrix().astype(np.float32)
        tprev = (rng.standard_normal(3) + 3).astype(np.float32)
        out = []
        for fn in (solve_lib.kts_update, solve_lib.kts_update_fast):
            res = Rt.copy().reshape(-1); Rc = np.zeros(9, np.float32); tc = np.zeros(3, np.float32)
            fn(_p(np.ascontiguousarray(A)), _p(b), _p(res), _p(np.ascontiguousarray(Rprev)), _p(tprev), _p(Rc), _p(tc))
            out.append((res.copy(), Rc.copy(), tc.copy()))
        assert np.abs(out[0][0][:12] - out[1][0][:12]).max() < 1e-15
        assert (out[1][0][12:] == np.array([0, 0, 0, 1.0])).all()
        worst = max(worst, np.abs(out[0][1] - out[1][1]).max(), np.abs(out[0][2] - out[1][2]).max())
    assert worst <= 2.4e-7 * 4                     # at most one float ulp of a pose entry (|t| < 4)
