"""Map deformation on the GPU (kt_deform.cu, kt_deform_map) against the FP64 restatement in oracle/deform_oracle.py.

Tolerances: node ids identical and weights within 1e-12 relative (both compute the same float / FP64 operations without FMA);
positions 1e-5 m and normals 1e-5 (the device solves the normal equations by a banded Cholesky in its own summation order, the oracle
by scipy's sparse LU).  The early-out decision and the number of Gauss-Newton steps must agree."""
import os
import sys

import numpy as np
import pytest

from conftest import ROOT

sys.path.insert(0, ROOT)
from oracle import deform_oracle as D  # noqa: E402

pytestmark = pytest.mark.gpu


def _dev(a):
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.uint8).reshape(-1).copy()).cuda()


def _host(t, dtype, shape):
    return t.cpu().numpy().view(dtype).reshape(shape)


def _records(v, nrm, kind, seed=0):
    from kintinuous_b200.binding import POINT_NORMAL_DTYPE, MESH_VERTEX_DTYPE
    rng = np.random.default_rng(seed)
    r = np.zeros(len(v), POINT_NORMAL_DTYPE if kind == 0 else MESH_VERTEX_DTYPE)
    for i, c in enumerate("xyz"):
        r[c] = v[:, i]; r["n" + c] = nrm[:, i]
    for c in ("r", "g", "b", "a"):
        r[c] = rng.integers(0, 256, len(v))
    if kind == 0:
        r["_p0"] = 1.0; r["curvature"] = rng.random(len(v)).astype(np.float32)
    return r


def _run_ops(kb, node_pos, node_times, con_src, con_t, con_dst, recs, vt, kind):
    import torch
    n = len(node_pos)
    npos = _dev(np.asarray(node_pos, np.float32)); nt = _dev(np.asarray(node_times, np.uint64))
    npos_t = npos.view(torch.float32).view(n, 3)
    m = len(con_src)
    cs = _dev(np.asarray(con_src, np.float32)); ct = _dev(np.asarray(con_t, np.uint64))
    cids = torch.zeros(m * 16, dtype=torch.uint8, device="cuda"); cw = torch.zeros(m * 32, dtype=torch.uint8, device="cuda")
    kb.ops.deform_weights(npos_t, nt, cs, 2, ct.view(torch.int64), cids, cw)
    params = torch.zeros(n * 12, dtype=torch.float64, device="cuda")
    rep = kb.ops.deform_optimise(npos_t, cs.view(torch.float32).view(m, 3), _dev(np.asarray(con_dst, np.float64)), cids, cw, params)
    N = len(recs)
    pin = _dev(recs); pout = torch.zeros_like(pin); vtd = _dev(np.asarray(vt, np.uint64))
    ids = torch.zeros(N * 16, dtype=torch.uint8, device="cuda"); w = torch.zeros(N * 32, dtype=torch.uint8, device="cuda")
    kb.ops.deform_weights(npos_t, nt, pin, kind, vtd.view(torch.int64), ids, w)
    kb.ops.deform_apply(npos_t, params, ids, w, pin, pout, kind, N)
    torch.cuda.synchronize()
    return (rep, _host(cids, np.int32, (m, 4)), _host(cw, np.float64, (m, 4)), params.cpu().numpy().reshape(n, 12),
            _host(ids, np.int32, (N, 4)), _host(w, np.float64, (N, 4)), pout.cpu().numpy().view(recs.dtype))


def _xyz(r, pre=""):
    return np.stack([r[pre + "x"], r[pre + "y"], r[pre + "z"]], -1).astype(np.float64)


def _check_against_oracle(node_pos, node_times, cs, ct, cd, recs, vt, kind, got, label):
    rep, cids, cw, x, ids, w, out = got
    wids, ww = D.weights(node_pos, node_times, cs, ct)
    assert np.array_equal(cids, wids) and np.abs(cw - ww).max() <= 1e-12, label
    vids, vw = D.weights(node_pos, node_times, _xyz(recs).astype(np.float32), vt)
    assert np.array_equal(ids, vids), label
    assert (np.abs(w - vw) <= 1e-12 * np.abs(vw)).all(), label
    ox, orep = D.Graph(node_pos, cs, cd, wids, ww).optimise()
    assert (rep.deformed, rep.iterations, rep.band) == (orep["deformed"], orep["iterations"], orep["band"]), (label, rep.as_dict(), orep)
    assert rep.solver_failed == 0
    p, nn = D.apply(node_pos, ox, vids, vw, _xyz(recs), _xyz(recs, "n"))
    dp = np.abs(_xyz(out) - p).max(); dn = np.abs(_xyz(out, "n") - nn).max()
    print(f"{label}: {rep.as_dict()}; |x - x_oracle| {np.abs(x - ox).max():.2e}, position {dp:.2e} m, normal {dn:.2e}")
    assert dp <= 1e-5 and dn <= 1e-5, label
    keep = [f for f in recs.dtype.names if f not in ("x", "y", "z", "nx", "ny", "nz")]
    for f in keep:
        assert np.array_equal(out[f], recs[f]), (label, f)
    return rep


def test_operators_match_the_oracle(built):
    import kintinuous_b200 as kb
    times, pos, vt, v, nrm = D.synthetic(7, 4000, 1_000_000)
    take = D.sample_nodes(pos, 0.2)
    node_pos, node_times = pos[take], times[take]
    assert 200 <= len(take) <= 1000
    assert (vt < node_times[0]).any() and (vt > node_times[-1]).any()
    # 4000 poses + 6000 point constraints = 10^4
    tf = (times - times[0]) / float(times[-1] - times[0])
    WR, Wt = D.warp(tf, 20.0, (3.0, -1.0, 2.0))
    corr = np.einsum("nij,nj->ni", WR, pos.astype(np.float64)) + Wt
    pi = np.random.default_rng(2).integers(0, len(v), 6000)
    ptf = np.clip((vt[pi].astype(np.float64) - times[0]) / float(times[-1] - times[0]), 0, 1)
    PR, Pt = D.warp(ptf, 20.0, (3.0, -1.0, 2.0))
    cs = np.concatenate([pos, v[pi]]); ct = np.concatenate([times, vt[pi]])
    cd = np.concatenate([corr, np.einsum("nij,nj->ni", PR, v[pi].astype(np.float64)) + Pt])
    for kind in (0, 1):
        recs = _records(v, nrm, kind)
        got = _run_ops(kb, node_pos, node_times, cs, ct, cd, recs, vt, kind)
        rep = _check_against_oracle(node_pos, node_times, cs, ct, cd, recs, vt, kind, got, f"warp kind {kind}")
        assert rep.deformed == 1 and rep.iterations >= 2
        again = _run_ops(kb, node_pos, node_times, cs, ct, cd, recs, vt, kind)
        assert again[3].tobytes() == got[3].tobytes() and again[6].tobytes() == got[6].tobytes()     # bitwise deterministic
    # identity: the early-out, the same decision as the oracle
    recs = _records(v[:10000], nrm[:10000], 0)
    got = _run_ops(kb, node_pos, node_times, pos, times, pos.astype(np.float64), recs, vt[:10000], 0)
    rep = _check_against_oracle(node_pos, node_times, pos, times, pos.astype(np.float64), recs, vt[:10000], 0, got, "identity")
    assert rep.deformed == 0 and rep.iterations == 0


def test_band_of_exactly_19_blocks(built):
    import kintinuous_b200 as kb
    # 19 nodes per turn of a shallow helix: node j and j + 19 nearly coincide, and a point at the time of node j + 19 next to them
    # takes both -- a term spanning 19 blocks of J^T J
    n = 120
    a = 2 * np.pi * np.arange(n) / 19
    node_pos = np.stack([np.cos(a), 0.002 * np.arange(n), np.sin(a)], 1).astype(np.float32)
    node_times = (1000 + 1000 * np.arange(n)).astype(np.uint64)
    rng = np.random.default_rng(4)
    j = rng.integers(0, n - 19, 400)
    cs = (node_pos[j] + node_pos[j + 19]) / 2 + rng.normal(0, 0.003, (400, 3)).astype(np.float32)
    ct = node_times[j + 19]
    cd = cs.astype(np.float64) * 1.5 + np.array([2.0, 0.5, -1.0])
    v = (node_pos[rng.integers(0, n, 50000)] + rng.normal(0, 0.2, (50000, 3))).astype(np.float32)
    vt = rng.integers(0, 130_000, 50000).astype(np.uint64)
    nrm = rng.normal(size=(50000, 3)).astype(np.float32)
    recs = _records(v, nrm, 0)
    got = _run_ops(kb, node_pos, node_times, cs, ct, cd, recs, vt, 0)
    rep = _check_against_oracle(node_pos, node_times, cs, ct, cd, recs, vt, 0, got, "band 19")
    assert rep.band == 19 and rep.deformed == 1


def test_singular_band_leaves_the_map_undeformed(built):
    import kintinuous_b200 as kb
    # Nodes and constraint sources exactly on the x axis: no term but E_rot touches R[2, 1] and R[1, 2], and E_rot's row c1 . c2 weighs
    # them equally at the identity, so J^T J is singular (rotation about the line is free) and a pivot of the first step is exactly 0.
    n = 30
    node_pos = np.zeros((n, 3), np.float32); node_pos[:, 0] = 0.1 * np.arange(n)
    node_times = (1000 + 1000 * np.arange(n)).astype(np.uint64)
    cs = np.zeros((2 * n, 3), np.float32); cs[:, 0] = 0.05 * np.arange(2 * n)
    ct = (1000 + 500 * np.arange(2 * n)).astype(np.uint64)
    cd = cs.astype(np.float64) + np.array([0.5, 1.0, 2.0])
    wids, ww = D.weights(node_pos, node_times, cs, ct)
    J = D.Graph(node_pos, cs, cd, wids, ww).jacobian(D.Graph.identity(n)).toarray()
    assert np.linalg.matrix_rank(J.T @ J) < 12 * n                                      # the oracle agrees: singular
    rng = np.random.default_rng(6)
    v = (node_pos[rng.integers(0, n, 2000)] + rng.normal(0, 0.3, (2000, 3))).astype(np.float32)
    nrm = rng.normal(size=(2000, 3)).astype(np.float32)
    vt = rng.integers(0, 32_000, 2000).astype(np.uint64)
    recs = _records(v, nrm, 0)
    rep, cids, cw, x, ids, w, out = _run_ops(kb, node_pos, node_times, cs, ct, cd, recs, vt, 0)
    print("singular:", rep.as_dict())
    assert (rep.solver_failed, rep.deformed, rep.iterations) == (1, 0, 1)
    assert np.array_equal(x, D.Graph.identity(n))                                        # the identity, not a partial step
    assert np.array_equal(_xyz(out), _xyz(recs))
    nn = _xyz(recs, "n"); nn /= np.linalg.norm(nn, axis=1, keepdims=True)
    assert np.abs(_xyz(out, "n") - nn).max() <= 1e-6
    for f in ("r", "g", "b", "a", "curvature", "_p0"):
        assert np.array_equal(out[f], recs[f])


def test_non_finite_constraints_are_rejected(built):
    import kintinuous_b200 as kb
    import torch
    n = 30
    node_pos = np.stack([0.1 * np.arange(n), 0.02 * np.sin(np.arange(n)), 0.03 * np.cos(np.arange(n))], 1).astype(np.float32)
    npos = _dev(node_pos).view(torch.float32).view(n, 3)
    cs = node_pos[::3].copy(); m = len(cs)
    cd = cs.astype(np.float64) + 1.0; cd[4, 2] = np.nan
    ids = _dev(np.tile(np.arange(4, dtype=np.int32), (m, 1)))
    w = _dev(np.full((m, 4), 0.25))
    params = torch.zeros(n * 12, dtype=torch.float64, device="cuda")
    with pytest.raises(kb.KtError, match="error -1.*not finite"):
        kb.ops.deform_optimise(npos, _dev(cs).view(torch.float32).view(m, 3), _dev(cd), ids, w, params)


# ---- the tracker ------------------------------------------------------------------------------------------------------------
ROWS, COLS, V, FRAMES = 240, 320, 256, 60


def _track(kb, n=FRAMES, deform_at=None, corrected=None):
    from kintinuous_b200 import synth
    trk = kb.Tracker(kb.Config.default(rows=ROWS, cols=COLS, vol=V, odometry=0, voxel_shift=2))
    trk.set_slice_processing(True, 8)
    trk.set_slice_meshing(True, 8)
    poses = []
    for k in range(n):
        if deform_at is not None and k == deform_at:
            dp = [trk.dense_pose(i) for i in range(trk.num_dense_poses())]
            trk.deform_map([(t, corrected(t, p)) for t, p, _ in dp], node_spacing=0.05)
        d, c = synth.render(k, COLS, ROWS)
        poses.append(bytes(trk.process_frame(d, c, k)))
    trk.finalise()
    return trk, poses


def _map(trk, getter_p, getter_m):
    P = [getter_p(i) for i in range(trk.num_slices())]
    M = [getter_m(i) for i in range(trk.num_slices())]
    return P, M


def _dense(trk):
    dp = [trk.dense_pose(i) for i in range(trk.num_dense_poses())]
    return np.array([t for t, _, _ in dp], np.uint64), np.array([p[:3, 3] for _, p, _ in dp], np.float32), dp


def _oracle_map(trk, corr_fn, spacing):
    """The oracle over the tracker's own slices and dense poses."""
    times, pos, dp = _dense(trk)
    corr = np.array([corr_fn(t, p)[:3, 3] for t, p, _ in dp], np.float32).astype(np.float64)     # kt_dense_pose is float
    out = {}
    for kind, get in ((0, trk.get_processed_slice), (1, lambda i: trk.get_slice_mesh(i)[0])):
        recs = [get(i) for i in range(trk.num_slices())]
        ut = np.concatenate([np.full(len(r), trk.slice_info(i).utime, np.uint64) for i, r in enumerate(recs)])
        allr = np.concatenate(recs)
        p, n, rep, *_ = D.deform(times, pos, times, corr, spacing, _xyz(allr).astype(np.float32), _xyz(allr, "n").astype(np.float32), ut)
        out[kind] = (allr, p, n, rep)
    return out


def _rigid():
    from scipy.spatial.transform import Rotation
    R = Rotation.from_rotvec([0.05, 0.25, -0.04]).as_matrix(); T = np.array([0.4, -0.25, 0.5])
    return R, T


def test_tracker_rigid_and_warp(built, tmp_path):
    """Rigid corrections T pose: the deformed map equals the oracle's within 1e-5 m, and is as close to T v as the oracle's.  That is
    looser than T v within 1e-5 m: the reference's stopping rule (error < 1e-3) ends Gauss-Newton after 2 steps on this 13-node,
    60-constraint graph, 1.76e-3 m short of T v on the farthest vertices, on the device and in the FP64 oracle alike."""
    import kintinuous_b200 as kb
    trk, _ = _track(kb)
    n = trk.num_slices()
    assert n >= 4
    R, T = _rigid()

    def rigid(t, p):
        q = np.eye(4); q[:3, :3] = R @ p[:3, :3]; q[:3, 3] = R @ p[:3, 3] + T
        return q
    rep = trk.deform_map([(t, rigid(t, p)) for t, p, _ in _dense(trk)[2]], node_spacing=0.05)
    print("rigid:", rep.as_dict())
    assert rep.deformed == 1 and rep.nodes >= 5
    P, M = _map(trk, trk.get_deformed_slice, trk.get_deformed_slice_mesh)
    ora = _oracle_map(trk, rigid, 0.05)
    for kind, got in ((0, np.concatenate(P)), (1, np.concatenate(M))):
        allr, p, nn, orep = ora[kind]
        assert orep["iterations"] == rep.iterations
        g = _xyz(got)
        want = _xyz(allr) @ R.T + T
        own = np.abs(p - want).max()
        err = np.abs(g - want).max()
        print(f"rigid kind {kind}: {len(g)} vertices, |deformed - T v| max {err:.2e} m (oracle's own {own:.2e}), vs oracle {np.abs(g - p).max():.2e}")
        assert np.abs(g - p).max() <= 1e-5 and np.abs(_xyz(got, "n") - nn).max() <= 1e-5
        assert err <= max(1e-5, own + 1e-5)
        if kind == 1:
            # distance to the analytic scene, moved by T, equals the undeformed map's distance to the scene
            from test_gpu_mesh import _scene_distance
            back = (g - T) @ R
            d0 = _scene_distance(_xyz(allr)); d1 = _scene_distance(back)
            assert np.abs(d1 - d0).max() <= err + 1e-6                     # the distance is 1-Lipschitz
    # the deformed PLY round-trips
    path = str(tmp_path / "deformed.ply")
    trk.save_deformed_mesh_ply(path)
    blob = open(path, "rb").read()
    head, body = blob.split(b"end_header\n", 1)
    nv = int([ln for ln in head.decode().splitlines() if ln.startswith("element vertex")][0].split()[-1])
    vdt = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4"), ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    pv = np.frombuffer(body, vdt, nv)
    allm = np.concatenate(M)
    assert nv == len(allm) and all(np.array_equal(pv[a], allm[b]) for a, b in (("x", "x"), ("y", "y"), ("z", "z"), ("nx", "nx"), ("red", "r")))
    ref = str(tmp_path / "mesh.ply"); trk.save_mesh_ply(ref)
    assert len(open(ref, "rb").read()) == len(blob)

    # a time-varying correction W(t)
    times = _dense(trk)[0]
    t0, t1 = float(times[0]), float(times[-1])

    def warp(t, p):
        Wr, Wt = D.warp(np.array((t - t0) / (t1 - t0)), 2.0, (0.15, -0.05, 0.15))
        q = np.eye(4); q[:3, :3] = Wr @ p[:3, :3]; q[:3, 3] = Wr @ p[:3, 3] + Wt
        return q
    rep = trk.deform_map([(t, warp(t, p)) for t, p, _ in _dense(trk)[2]], node_spacing=0.05)
    print("warp:", rep.as_dict())
    assert rep.deformed == 1
    P, M = _map(trk, trk.get_deformed_slice, trk.get_deformed_slice_mesh)
    ora = _oracle_map(trk, warp, 0.05)
    for kind, got in ((0, np.concatenate(P)), (1, np.concatenate(M))):
        allr, p, nn, orep = ora[kind]
        assert (orep["iterations"], orep["deformed"]) == (rep.iterations, rep.deformed)
        g = _xyz(got)
        assert np.abs(g - p).max() <= 1e-5 and np.abs(_xyz(got, "n") - nn).max() <= 1e-5
        ut = np.concatenate([np.full(len(r), trk.slice_info(i).utime, np.uint64) for i, r in enumerate(P if kind == 0 else M)])
        Wr, Wt = D.warp((ut.astype(np.float64) - t0) / (t1 - t0), 2.0, (0.15, -0.05, 0.15))
        res = np.linalg.norm(g - (np.einsum("nij,nj->ni", Wr, _xyz(allr)) + Wt), axis=1)
        ores = np.linalg.norm(p - (np.einsum("nij,nj->ni", Wr, _xyz(allr)) + Wt), axis=1)
        q = np.quantile(res, [0.5, 0.9, 0.99, 1.0])
        print(f"warp kind {kind}: residual to W(t) v: median {q[0]:.2e}, 90 % {q[1]:.2e}, 99 % {q[2]:.2e}, max {q[3]:.2e} m "
              f"(oracle's own max {ores.max():.2e})")
        assert res.max() <= ores.max() + 1e-5
    trk.close()


def test_non_interference_and_errors(built):
    import kintinuous_b200 as kb
    ref, ref_poses = _track(kb)
    R, T = _rigid()

    def rigid(t, p):
        q = np.eye(4); q[:3, :3] = R @ p[:3, :3]; q[:3, 3] = R @ p[:3, 3] + T
        return q
    mid, mid_poses = _track(kb, deform_at=FRAMES // 2, corrected=rigid)
    assert mid_poses == ref_poses
    n = ref.num_slices()
    assert mid.num_slices() == n
    from test_gpu_mesh import _canon
    for i in range(n):
        assert np.array_equal(_canon(ref.get_slice(i)[0]), _canon(mid.get_slice(i)[0]))     # extraction order is unspecified (atomics)
        assert ref.get_processed_slice(i).tobytes() == mid.get_processed_slice(i).tobytes()
        a, b = ref.get_slice_mesh(i), mid.get_slice_mesh(i)
        assert a[0].tobytes() == b[0].tobytes() and np.array_equal(a[1], b[1])
    assert [mid.dense_pose(i)[1].tobytes() for i in range(mid.num_dense_poses())] == [ref.dense_pose(i)[1].tobytes() for i in range(ref.num_dense_poses())]
    # slices recorded after the call
    covered = len([1 for i in range(n) if mid.slice_info(i).utime < FRAMES // 2])
    with pytest.raises(kb.KtError, match="error -3"):
        mid.get_deformed_slice(n - 1)
    with pytest.raises(kb.KtError, match="error -3"):
        mid.get_deformed_slice_mesh(n - 1)
    assert covered >= 1
    mid.get_deformed_slice(0)
    mid.close()

    # identity corrections: the original bytes, deformed == 0
    dp = _dense(ref)[2]
    rep = ref.deform_map([(t, p) for t, p, _ in dp], node_spacing=0.05)
    assert rep.deformed == 0 and rep.iterations == 0
    for i in range(n):
        assert ref.get_deformed_slice(i).tobytes() == ref.get_processed_slice(i).tobytes()
        assert ref.get_deformed_slice_mesh(i).tobytes() == ref.get_slice_mesh(i)[0].tobytes()
    # errors
    with pytest.raises(kb.KtError, match="error -1"):
        ref.deform_map([(12345678, dp[0][1])], node_spacing=0.05)                       # not a dense pose timestamp
    with pytest.raises(kb.KtError, match="error -1.*not finite"):
        ref.deform_map([(t, p) for t, p, _ in dp], points=[(dp[3][0], (np.nan, 0.0, 1.0), (0.0, 0.0, 1.0))], node_spacing=0.05)
    bad = dp[5][1].copy(); bad[1, 3] = np.inf
    with pytest.raises(kb.KtError, match="error -1.*not finite"):
        ref.deform_map([(dp[5][0], bad)], node_spacing=0.05)
    with pytest.raises(kb.KtError, match="node_spacing"):
        ref.deform_map([(t, p) for t, p, _ in dp], node_spacing=10.0)                    # fewer than k + 1 nodes
    import ctypes as C
    from kintinuous_b200.binding import POINT_NORMAL_DTYPE
    buf = np.zeros(1, POINT_NORMAL_DTYPE); cnt = C.c_size_t(0)
    i_big = max(range(n), key=lambda i: len(ref.get_processed_slice(i)))
    ref.lib.kt_get_deformed_slice(ref.h, i_big, buf.ctypes.data_as(C.c_void_p), C.c_size_t(1), C.byref(cnt))
    assert cnt.value == len(ref.get_processed_slice(i_big)) and buf.tobytes() == ref.get_processed_slice(i_big)[:1].tobytes()
    ref.reset()
    with pytest.raises(kb.KtError, match="error -3"):
        ref.deform_map([], node_spacing=0.05)                                            # nothing recorded
    with pytest.raises(kb.KtError, match="error -3"):
        ref.save_deformed_mesh_ply(os.devnull)
    ref.close()
