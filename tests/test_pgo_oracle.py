"""Loop closure's pose-graph restatement (oracle/pgo_oracle.py) and the host logic of kt_pgo.hpp, without a GPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from conftest import ROOT
from oracle import pgo_oracle as P


@pytest.fixture(scope="module")
def lib():
    out = os.path.join(ROOT, "tests", "cpp", "_build")
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, "libkt_pgo_host.so")
    src = os.path.join(ROOT, "tests", "cpp", "pgo_host.cpp")
    hdrs = [os.path.join(ROOT, "kintinuous_b200", "csrc", h) for h in ("kt_pgo.hpp", "kt_deform.hpp", "kt_posegraph.hpp")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in [src] + hdrs):
        subprocess.check_call(["g++", "-std=c++14", "-O2", "-shared", "-fPIC", "-I", os.path.join(ROOT, "kintinuous_b200", "csrc"), "-o", so, src])
    lib = C.CDLL(so)
    lib.kth_wrap.restype = C.c_double
    lib.kth_wrap.argtypes = [C.c_double]
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _random_poses(rng, n, scale=2.0):
    R = Rotation.from_rotvec(rng.normal(0, 0.8, (n, 3))).as_matrix()
    X = np.zeros((n, 4, 4)); X[:, :3, :3] = R; X[:, :3, 3] = rng.normal(0, scale, (n, 3)); X[:, 3, 3] = 1
    return X


def test_jacobians_match_central_differences():
    rng = np.random.default_rng(1)
    X = _random_poses(rng, 6)
    fi = np.array([-1, 0, 1, 2, 4]); fj = np.array([0, 1, 3, 5, 2])
    fz = np.concatenate([P.vector(X[:1]) + 0.01, rng.normal(0, 0.3, (4, 6))])
    e, Ji, Jj = P.linearise(X, fi, fj, fz)
    h = 1e-6
    for node, J in (("j", Jj), ("i", Ji)):
        for c in range(6):
            d = np.zeros((len(X), 6))
            for f in range(len(fi)):
                k = fj[f] if node == "j" else fi[f]
                if k < 0:
                    continue
                d[:] = 0; d[k, c] = h
                ep = P.linearise(P.update(X, d), fi[f:f + 1], fj[f:f + 1], fz[f:f + 1])[0][0]
                em = P.linearise(P.update(X, -d), fi[f:f + 1], fj[f:f + 1], fz[f:f + 1])[0][0]
                num = (ep - em) / (2 * h)
                assert np.abs(num - J[f, :, c]).max() <= 1e-5 * max(1.0, np.abs(num).max()), (node, f, c, num, J[f, :, c])


def test_euler_and_wrap_round_trip(lib):
    rng = np.random.default_rng(2)
    v = np.stack([rng.uniform(-np.pi, np.pi, 500), rng.uniform(-1.5, 1.5, 500), rng.uniform(-np.pi, np.pi, 500)], 1)
    R = P.rot(v)
    assert np.abs(P.ypr(R) - v).max() <= 1e-12
    assert np.abs(R @ np.swapaxes(R, 1, 2) - np.eye(3)).max() <= 1e-14
    for k in range(20):
        Rk = np.ascontiguousarray(R[k]); out = np.zeros(3); lib.kth_ypr(_p(Rk), _p(out))
        assert np.abs(out - v[k]).max() <= 1e-12
        Rb = np.zeros(9); vk = np.ascontiguousarray(v[k]); lib.kth_rot(_p(vk), _p(Rb))
        assert np.abs(Rb.reshape(3, 3) - R[k]).max() <= 1e-15
    a = np.concatenate([rng.uniform(-20, 20, 1000), [np.pi, -np.pi, 0.0, 3 * np.pi, -3 * np.pi]])
    w = P.wrap(a)
    assert ((w > -np.pi) & (w <= np.pi)).all()
    assert np.abs(np.sin(w) - np.sin(a)).max() <= 1e-12 and np.abs(np.cos(w) - np.cos(a)).max() <= 1e-12
    assert w[-5] == np.pi and w[-4] == np.pi
    assert all(lib.kth_wrap(float(x)) == float(y) for x, y in zip(a, w))
    X = _random_poses(rng, 10)
    assert np.abs(P.pose(P.vector(X)) - X).max() <= 1e-12
    Pf = X.astype(np.float32)
    assert np.abs(P.from_isam(P.to_isam(Pf)) - Pf.astype(np.float64)).max() == 0.0


def _chain(n, loops, X0):
    fi, fj, fz = P.chain_factors(X0, loops)
    return fi, fj, fz


def test_consistent_loop_returns_the_tracked_poses():
    # translations on a dyadic grid and identity rotations: every float operation of the measurement path is exact
    rng = np.random.default_rng(3)
    n = 40
    X = np.tile(np.eye(4), (n, 1, 1)); X[:, :3, 3] = np.cumsum(rng.integers(-8, 9, (n, 3)) / 16.0, 0)
    Pw = P.from_isam(X).astype(np.float32)
    C = np.linalg.inv(Pw[30].astype(np.float64)) @ Pw[3].astype(np.float64)
    times = np.arange(n, dtype=np.uint64) * 10 + 5
    take, Xo, rep, acc = P.close_loop(times, Pw, [(times[30], times[3], C)])
    assert acc and rep["chi2_initial"] <= 1e-20 and rep["chi2_final"] <= 1e-20
    assert np.abs(Xo - Pw.astype(np.float64)).max() <= 1e-9


def test_drifted_circle_is_corrected():
    """Drift of 0.1 m over 2000 poses; one exact loop from the last pose to the first closes it: the last pose ends within 1 cm of
    ground truth and no pose is further from it than before."""
    Xgt, Xd, _ = P.synthetic_chain(4, 2000, 0)
    n = len(Xgt)
    loops = [(n - 1, 0, P.vector(np.linalg.inv(Xgt[n - 1]) @ Xgt[0]))]
    fi, fj, fz = P.chain_factors(Xd, loops)
    X, rep = P.optimise(Xd, fi, fj, fz)
    d0 = np.linalg.norm(Xd[:, :3, 3] - Xgt[:, :3, 3], axis=1); d = np.linalg.norm(X[:, :3, 3] - Xgt[:, :3, 3], axis=1)
    print(rep, f"drift max {d0.max():.3f} m, end {d0[-1]:.3f} m -> max {d.max():.3f} m, end {d[-1]:.4f} m")
    assert rep["solver_failed"] == 0 and 2 <= rep["iterations"] < 100 and rep["chi2_final"] < rep["chi2_initial"]
    assert d0[-1] > 0.05 and d[-1] <= 0.01 and d.max() <= d0.max()
    assert np.abs(P.vector(np.linalg.inv(X[n - 1]) @ X[0]) - loops[0][2]).max() <= 1e-3


def test_prior_anchor_is_equivariant():
    Xgt, Xd, loops = P.synthetic_chain(5, 300, 2)
    fi, fj, fz = P.chain_factors(Xd, loops)
    X, rep = P.optimise(Xd, fi, fj, fz)
    G = P.pose(np.array([1.0, -2.0, 0.5, 0.7, -0.2, 0.3]))
    Xg = G @ Xd
    fig, fjg, fzg = P.chain_factors(Xg, loops)
    assert np.abs(fzg[1:] - fz[1:]).max() <= 1e-9                       # relative measurements do not move
    X2, rep2 = P.optimise(Xg, fig, fjg, fzg)
    assert rep2["iterations"] == rep["iterations"] and abs(rep2["chi2_final"] - rep["chi2_final"]) <= 1e-9 * max(1.0, rep["chi2_final"])
    assert np.abs(X2 - G @ X).max() <= 1e-9


def test_node_selection(lib):
    rng = np.random.default_rng(6)
    n = 400
    pos = np.cumsum(rng.normal(0, 0.02, (n, 3)), 0).astype(np.float32)
    flagged = np.zeros(n, np.uint8); flagged[[17, 250]] = 1
    for spacing in (0.0, 0.05, 0.2):
        want = P.select_nodes(pos, flagged.astype(bool), spacing)
        out = np.zeros(n, np.int32)
        k = lib.kth_select_nodes(_p(pos), _p(flagged), C.c_size_t(n), C.c_float(spacing), _p(out))
        assert np.array_equal(out[:k], want), spacing
        assert want[0] == 0 and want[-1] == n - 1 and 17 in want and 250 in want
        if spacing == 0.0:
            assert len(want) == n
        else:
            last = 0
            for i in range(1, n - 1):               # the -fl rule, literally
                d = np.float32(np.linalg.norm(pos[i] - pos[last]))
                if abs(float(d) - spacing) > 1e-6:
                    assert (i in want) == (d > spacing or flagged[i]), (spacing, i)
                if i in want:
                    last = i


def test_measurements_match_the_host_bit_for_bit(lib):
    rng = np.random.default_rng(7)
    for _ in range(200):
        A = _random_poses(rng, 2).astype(np.float32)
        z = np.zeros(6); lib.kth_odometry_z(_p(np.ascontiguousarray(A[0])), _p(np.ascontiguousarray(A[1])), _p(z))
        assert z.tobytes() == P.odometry_z(A[0], A[1]).tobytes()
        Cm = np.ascontiguousarray(_random_poses(rng, 1)[0])
        zl = np.zeros(6); lib.kth_loop_z(_p(Cm), _p(zl))
        assert np.abs(zl - P.loop_z(Cm)).max() <= 1e-15
        Xh = np.zeros(16); lib.kth_pose_to_isam(_p(np.ascontiguousarray(A[0])), _p(Xh))
        assert Xh.tobytes() == P.to_isam(A[0]).reshape(-1).tobytes()
    # the float measurement equals the FP64 relative pose to float precision
    A = _random_poses(rng, 2).astype(np.float32)
    Xa = P.to_isam(A)
    assert np.abs(P.odometry_z(A[0], A[1]) - P.vector(np.linalg.inv(Xa[0]) @ Xa[1])).max() <= 1e-5


def test_invalid_constraints_are_rejected(lib):
    good = np.eye(4); good[:3, 3] = [0.1, 0.2, 0.3]
    bad_nan = good.copy(); bad_nan[1, 3] = np.nan
    bad_rot = good.copy(); bad_rot[0, 0] = 1.01
    for Cm, want in ((good, 0), (bad_nan, 1), (bad_rot, 2)):
        assert P.check_constraint(Cm) == want
        assert lib.kth_check_constraint(_p(np.ascontiguousarray(Cm))) == want
    times = np.arange(10, dtype=np.uint64)
    poses = np.tile(np.eye(4, dtype=np.float32), (10, 1, 1))
    with pytest.raises(KeyError):
        P.close_loop(times, poses, [(99, 2, good)])


def test_plan_levels(lib):
    for n, loops in ((2, []), (1000, [(900, 10)]), (1 << 14, [(i * 200 + 7, i * 200 + 8) for i in range(64)]), (1 << 18, [(70000, 64), (128, 129)])):
        li = np.array([l[0] for l in loops], np.int32); lj = np.array([l[1] for l in loops], np.int32)
        sizes = np.zeros(16, np.int32); ti = np.zeros(max(1, len(loops)), np.int32); tj = np.zeros_like(ti)
        nl = lib.kth_plan(n, len(loops), _p(li), _p(lj), _p(sizes), 16, _p(ti), _p(tj))
        s = list(sizes[:nl])
        assert s[0] == n and all(a > b for a, b in zip(s, s[1:]))
        assert s[-1] <= 2 * len(loops) + 3, s                          # the dense top: loop endpoints, first and last
        assert (ti[:len(loops)] != tj[:len(loops)]).all() and (ti[:len(loops)] < s[-1]).all()
