"""The deformation graph's CPU restatement (oracle/deform_oracle.py) and the host logic of kt_deform.hpp, without a GPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from conftest import ROOT
from oracle import deform_oracle as D


@pytest.fixture(scope="module")
def lib():
    out = os.path.join(ROOT, "tests", "cpp", "_build")
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, "libkt_deform_host.so")
    src = os.path.join(ROOT, "tests", "cpp", "deform_host.cpp")
    hdr = os.path.join(ROOT, "kintinuous_b200", "csrc", "kt_deform.hpp")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-std=c++14", "-O2", "-shared", "-fPIC", "-I", os.path.join(ROOT, "kintinuous_b200", "csrc"), "-o", so, src])
    lib = C.CDLL(so)
    lib.kth_pose_constraints.restype = C.c_long
    lib.kth_first_non_finite_f.restype = C.c_long
    lib.kth_first_non_finite_d.restype = C.c_long
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _problem(seed=1, n_poses=1500, n_verts=4000, spacing=0.2):
    times, pos, vt, v, nrm = D.synthetic(seed, n_poses, n_verts)
    return times, pos, vt, v, nrm, spacing


def test_jacobian_matches_finite_differences():
    times, pos, vt, v, nrm, spacing = _problem(n_poses=300, n_verts=10)
    take = D.sample_nodes(pos, spacing)
    npos, ntimes = pos[take], times[take]
    src = pos[::7]; st = times[::7]
    ids, w = D.weights(npos, ntimes, src, st)
    g = D.Graph(npos, src, src.astype(np.float64) + 0.3, ids, w)
    rng = np.random.default_rng(3)
    x = D.Graph.identity(g.n) + rng.normal(0, 0.05, (g.n, 12))
    J = g.jacobian(x).toarray()
    h = 1e-6
    fd = np.zeros_like(J)
    for c in range(12 * g.n):
        dx = np.zeros(12 * g.n); dx[c] = h
        fd[:, c] = (g.residual(x + dx.reshape(g.n, 12)) - g.residual(x - dx.reshape(g.n, 12))) / (2 * h)
    assert np.abs(J - fd).max() < 1e-6 * max(1.0, np.abs(J).max())


@pytest.mark.parametrize("rotvec,tol", [((0.0, 0.0, 0.0), 1e-9), ((0.1, 0.3, -0.05), 1e-5)])
def test_rigid_correction_is_reproduced(rotvec, tol):
    # With a rotation the reference's stopping rule (|delta| < 1e-2, error < 1e-3 or |d error| < 1e-5 error) ends Gauss-Newton
    # after 3 steps, a few micrometres short of T v; a pure translation is linear and is solved exactly.
    times, pos, vt, v, nrm, spacing = _problem()
    R = Rotation.from_rotvec(rotvec).as_matrix(); T = np.array([2.0, -1.0, 3.0])
    corr = pos.astype(np.float64) @ R.T + T
    p, n, rep, x, _, _ = D.deform(times, pos, times, corr, spacing, v, nrm, vt)
    assert rep["deformed"] == 1 and rep["iterations"] >= 1
    assert np.abs(p - (v.astype(np.float64) @ R.T + T)).max() < tol
    want_n = nrm.astype(np.float64) @ R.T
    l = np.linalg.norm(want_n, axis=1, keepdims=True)
    want_n = np.where(l > 0, want_n / np.where(l > 0, l, 1), 0)             # the float32 input normals are unit to ~1e-7
    assert np.abs(n - want_n).max() < 10 * tol
    assert (np.abs(n[::50]) == 0).all()                                   # zero normals stay zero


def test_identity_takes_the_early_out():
    times, pos, vt, v, nrm, spacing = _problem()
    p, n, rep, x, _, _ = D.deform(times, pos, times, pos.astype(np.float64), spacing, v, nrm, vt)
    assert rep["deformed"] == 0 and rep["iterations"] == 0 and rep["constraint_error"] < 0.1
    assert np.array_equal(p, v.astype(np.float64)) and np.array_equal(x, D.Graph.identity(len(x)))


def _brute_weights(npos, ntimes, v, t):
    """weightVerticesSeq written out literally for one vertex."""
    n = len(npos)
    f = D.nearest_node(ntimes, t)
    cand = []
    for j in range(f, -1, -1):
        cand.append(j)
        if len(cand) == D.LOOKBACK:
            break
    j = f + 1
    while len(cand) < D.LOOKBACK and j < n:
        cand.append(j); j += 1
    d = sorted((float(D._dist_f32(npos[j], v)), j) for j in cand)
    dmax = d[D.K][0]
    ws = [((1.0 - np.linalg.norm(v.astype(np.float64) - npos[j].astype(np.float64)) / dmax) ** 2, j) for _, j in d[:D.K]]
    s = sum(w for w, _ in ws)
    ws = sorted((j, w / s) for w, j in ws)
    return [j for j, _ in ws], [w for _, w in ws]


def test_weights():
    times, pos, vt, v, nrm, spacing = _problem(n_verts=3000)
    take = D.sample_nodes(pos, spacing)
    npos, ntimes = pos[take], times[take]
    ids, w = D.weights(npos, ntimes, v, vt)
    assert ids.shape == (len(v), D.K) and w.shape == (len(v), D.K)
    assert np.abs(w.sum(1) - 1).max() < 1e-12 and (w >= 0).all()
    assert ((ids.max(1) - ids.min(1)) <= 19).all() and (np.diff(ids, axis=1) > 0).all()
    for i in range(0, len(v), 7):
        bi, bw = _brute_weights(npos, ntimes, v[i], vt[i])
        assert list(ids[i]) == bi
        assert np.abs(w[i] - bw).max() <= 1e-12 * max(bw)


def test_times_outside_the_nodes_clamp(lib):
    times = np.array([100, 200, 300, 400, 500, 600], np.uint64)
    for t, want in [(0, 0), (99, 0), (100, 0), (149, 0), (150, 1), (151, 1), (600, 5), (601, 5), (10 ** 12, 5), (350, 3), (349, 2)]:
        assert D.nearest_node(times, t) == want, t
        assert lib.kth_nearest_node(_p(times), len(times), C.c_uint64(t)) == want, t
    assert list(D.nearest_nodes(times, np.array([0, 10 ** 12, 350, 351], np.uint64))) == [0, 5, 3, 3]
    rng = np.random.default_rng(5)
    nt = np.cumsum(rng.integers(1, 1000, 300)).astype(np.uint64)
    ts = rng.integers(0, int(nt[-1]) + 5000, 5000).astype(np.uint64)
    ts[:300] = nt
    vec = D.nearest_nodes(nt, ts)
    for t, f in zip(ts, vec):
        assert D.nearest_node(nt, t) == f == lib.kth_nearest_node(_p(nt), len(nt), C.c_uint64(int(t)))


def test_host_logic_equals_the_oracle(lib):
    times, pos, vt, v, nrm, spacing = _problem()
    for s in (0.0, 0.05, 0.2, 0.8):
        out = np.zeros(len(pos), np.int32)
        k = lib.kth_sample_nodes(_p(pos), C.c_size_t(len(pos)), C.c_float(s), _p(out))
        assert np.array_equal(out[:k], D.sample_nodes(pos, s)), s
    for n in (5, 6, 9, 40):
        off = np.zeros(n + 1, np.int32); nb = np.zeros(n * 8, np.int32)
        lib.kth_connect_seq(n, _p(off), _p(nb))
        want = D.connect_seq(n)
        assert [list(nb[off[i]:off[i + 1]]) for i in range(n)] == want
    sel = np.arange(0, len(times), 3)
    corr = pos[sel].astype(np.float64) + 0.5
    src = np.zeros((len(sel), 3), np.float32); dst = np.zeros((len(sel), 3))
    assert lib.kth_pose_constraints(_p(times), _p(pos), C.c_size_t(len(times)), _p(times[sel]), _p(corr), C.c_size_t(len(sel)), _p(src), _p(dst)) == -1
    ct, cs, cd = D.pose_constraints(times, pos, times[sel], corr)
    assert np.array_equal(src, cs) and np.array_equal(dst, cd)
    bad = times[sel].copy(); bad[4] = 7
    assert lib.kth_pose_constraints(_p(times), _p(pos), C.c_size_t(len(times)), _p(bad), _p(corr), C.c_size_t(len(sel)), _p(src), _p(dst)) == 4


def test_non_finite_vertices_keep_their_nodes_in_the_window(lib):
    # a NaN or infinite distance must never leave a slot of the k + 1 nearest unfilled (its id would index past the node table)
    rng = np.random.default_rng(8)
    for trial in range(300):
        n = int(rng.integers(5, 21)); lo = int(rng.integers(0, 1000))
        d = rng.random(n).astype(np.float32)
        kind = trial % 3
        if kind == 0:
            d[:] = np.nan
        elif kind == 1:
            d[rng.random(n) < 0.7] = np.inf
        else:
            d[rng.random(n) < 0.5] = np.nan
        bd = np.zeros(D.K + 1, np.float32); bi = np.zeros(D.K + 1, np.int32)
        lib.kth_select(_p(d), lo, n, _p(bd), _p(bi))
        assert ((bi >= lo) & (bi < lo + n)).all() and len(set(bi)) == D.K + 1, (d, bi)
        key = np.where(np.isnan(d), np.inf, d)
        want = lo + np.argsort(key, kind="stable")[:D.K + 1]                           # (distance, id), NaN as +inf
        assert list(bi) == list(want)
    # the oracle: vertices with NaN / infinite coordinates take nodes of their window, weights without NaN
    times, pos, vt, v, nrm, spacing = _problem(n_verts=300)
    take = D.sample_nodes(pos, spacing)
    npos, ntimes = pos[take], times[take]
    v = v.copy(); v[::3] = np.nan; v[1::3, 0] = np.inf
    ids, w = D.weights(npos, ntimes, v, vt)
    f = D.nearest_nodes(ntimes, vt); lo = np.maximum(f - 19, 0)
    assert ((ids >= lo[:, None]) & (ids < np.minimum(lo + 20, len(npos))[:, None])).all()
    assert np.isfinite(w).all() and np.abs(w.sum(1) - 1).max() < 1e-12


def test_non_finite_constraints_are_rejected(lib):
    for dt, fn in ((np.float32, lib.kth_first_non_finite_f), (np.float64, lib.kth_first_non_finite_d)):
        a = np.arange(12, dtype=dt)
        assert fn(_p(a), C.c_size_t(len(a))) == -1
        for bad in (np.nan, np.inf, -np.inf):
            b = a.copy(); b[7] = bad
            assert fn(_p(b), C.c_size_t(len(b))) == 7
    times, pos, vt, v, nrm, spacing = _problem(n_verts=10)
    corr = pos.astype(np.float64) + 1.0
    bad = corr.copy(); bad[5, 1] = np.nan
    with pytest.raises(ValueError):
        D.deform(times, pos, times, bad, spacing, v, nrm, vt)
    with pytest.raises(ValueError):
        D.deform(times, pos, times, corr, spacing, v, nrm, vt, points=(times[:2], np.array([[0, 0, np.nan], [1, 1, 1]], np.float32), corr[:2]))
