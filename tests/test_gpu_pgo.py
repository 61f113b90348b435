"""Loop closure on the GPU (kt_pgo.cu, kt_close_loop) against the FP64 restatement in oracle/pgo_oracle.py.

Tolerances: node poses 1e-9 (m and rotation entries) and chi2 1e-9 relative, with the same number of Gauss-Newton steps -- the
device eliminates the normal equations in its own order (segments, a dense top), the oracle uses a dense / sparse Cholesky."""
import sys

import numpy as np
import pytest

from conftest import ROOT

sys.path.insert(0, ROOT)
from oracle import pgo_oracle as P  # noqa: E402
from oracle import deform_oracle as D  # noqa: E402

pytestmark = pytest.mark.gpu


def _factors(fi, fj, fz):
    from kintinuous_b200.binding import PGO_FACTOR_DTYPE
    f = np.zeros(len(fi), PGO_FACTOR_DTYPE)
    f["i"] = fi; f["j"] = fj; f["z"] = fz
    return f


def _run(kb, X0, fi, fj, fz):
    import torch
    poses = torch.from_numpy(np.ascontiguousarray(X0, np.float64)).cuda()
    f = torch.from_numpy(_factors(fi, fj, fz).view(np.uint8)).cuda()
    out = torch.zeros_like(poses)
    rep = kb.ops.pgo_optimise(poses, f, out)
    torch.cuda.synchronize()
    return out.cpu().numpy(), rep


def _graph(seed, n, L):
    Xgt, Xd, loops = P.synthetic_chain(seed, n, L)
    if L >= 4:                                   # endpoints on fixed segment boundaries, and adjacent / shared endpoints
        loops[0] = (n - 64, 64, P.vector(np.linalg.inv(Xgt[n - 64]) @ Xgt[64]))
        loops[1] = (n - 63, 65, P.vector(np.linalg.inv(Xgt[n - 63]) @ Xgt[65]))
        loops[2] = (n - 64, 128, P.vector(np.linalg.inv(Xgt[n - 64]) @ Xgt[128]))
        loops[3] = (300, 301, P.vector(np.linalg.inv(Xgt[300]) @ Xgt[301]))
    return Xd, P.chain_factors(Xd, loops)


@pytest.mark.parametrize("n,L", [(1 << 10, 1), (1 << 10, 16), (1 << 12, 64), (1 << 14, 16), (1 << 16, 64), (1 << 18, 64)])
def test_operator_matches_the_oracle(built, n, L):
    import kintinuous_b200 as kb
    X0, (fi, fj, fz) = _graph(n + L, n, L)
    X, rep = _run(kb, X0, fi, fj, fz)
    Xo, orep = P.optimise(X0, fi, fj, fz)
    dX = np.abs(X - Xo).max()
    print(f"n={n} L={L}: {rep.as_dict()} oracle {orep}; |X - X_oracle| {dX:.2e}")
    assert rep.solver_failed == 0 and orep["solver_failed"] == 0
    assert rep.iterations == orep["iterations"] and rep.iterations >= 2 and rep.step_ms > 0
    assert (rep.nodes, rep.factors, rep.loops) == (n, n + L, L)
    assert dX <= 1e-9
    assert abs(rep.chi2_final - orep["chi2_final"]) <= 1e-9 * max(orep["chi2_final"], 1.0)
    assert abs(rep.chi2_initial - orep["chi2_initial"]) <= 1e-9 * orep["chi2_initial"]
    if n == 1 << 12:
        X2, rep2 = _run(kb, X0, fi, fj, fz)
        assert X2.tobytes() == X.tobytes() and rep2.chi2_final == rep.chi2_final          # bitwise deterministic


def test_singular_graph_fails_and_too_many_loops_are_refused(built):
    import kintinuous_b200 as kb
    # node 1 at pitch -90 degrees relative to node 0: yaw and roll are one direction there, G is infinite, the factorisation fails
    X0 = np.tile(np.eye(4), (40, 1, 1))
    X0[1:, :3, :3] = np.array([[0.0, 0.0, -1.0], [0.0, 1.0, 0.0], [1.0, 0.0, 0.0]])
    X0[:, 0, 3] = np.arange(40) * 0.1
    fi, fj, fz = P.chain_factors(X0, [(30, 2, P.vector(np.linalg.inv(X0[30]) @ X0[2]))])
    X, rep = _run(kb, X0, fi, fj, fz)
    Xo, orep = P.optimise(X0, fi, fj, fz)
    print("singular:", rep.as_dict(), orep)
    assert (rep.solver_failed, rep.iterations) == (1, 1) and (orep["solver_failed"], orep["iterations"]) == (1, 1)
    assert np.array_equal(X, X0)
    _, (fi, fj, fz) = _graph(9, 2000, 65)
    with pytest.raises(kb.KtError, match="error -4"):
        _run(kb, P.synthetic_chain(9, 2000, 0)[1], fi, fj, fz)


# ---- the tracker ----------------------------------------------------------------------------------------------------------------
ROWS, COLS, V, FRAMES = 240, 320, 256, 60
T1, T2 = 55, 5


def _track(kb, n=FRAMES, loop_at=None, loop_args=None):
    from kintinuous_b200 import synth
    trk = kb.Tracker(kb.Config.default(rows=ROWS, cols=COLS, vol=V, odometry=0, voxel_shift=2))
    trk.set_slice_processing(True, 8)
    trk.set_slice_meshing(True, 8)
    poses = []
    for k in range(n):
        if loop_at is not None and k == loop_at:
            trk.close_loop(*loop_args)
        d, c = synth.render(k, COLS, ROWS)
        poses.append(bytes(trk.process_frame(d, c, k)))
    trk.finalise()
    return trk, poses


def _gt(k):
    from kintinuous_b200 import synth
    R, t = synth.pose(k)
    G = np.eye(4); G[:3, :3] = R; G[:3, 3] = t
    return G


def _constraint(t1, t2, rotvec, shift):
    from scipy.spatial.transform import Rotation
    E = np.eye(4); E[:3, :3] = Rotation.from_rotvec(rotvec).as_matrix(); E[:3, 3] = shift
    return np.linalg.inv(_gt(t1)) @ _gt(t2) @ E


def _dense(trk):
    dp = [trk.dense_pose(i) for i in range(trk.num_dense_poses())]
    return np.array([t for t, _, _ in dp], np.uint64), np.array([p for _, p, _ in dp], np.float32)


def _inliers(seed, C, n=10):
    """n points in front of the camera at time1 and the same points seen from the camera at time2 (x2 = C^-1 x1), with noise."""
    rng = np.random.default_rng(seed)
    a = np.stack([rng.uniform(-1, 1, n), rng.uniform(-0.8, 0.8, n), rng.uniform(0.8, 2.5, n)], 1)
    b = a @ np.linalg.inv(C)[:3, :3].T + np.linalg.inv(C)[:3, 3] + rng.normal(0, 0.003, a.shape)
    return a.astype(np.float32), b.astype(np.float32)


def _expected_map(trk, take, Pn, loops, spacing):
    """deform_oracle over the tracker's slices with kt_close_loop's constraints built from the oracle's node poses."""
    times, poses = _dense(trk)
    at = {int(t): i for i, t in enumerate(times)}
    pt, ps, pd = [], [], []
    for k, idx in enumerate(take):
        pt.append(times[idx]); ps.append(poses[idx][:3, 3]); pd.append(Pn[k][:3, 3])
    node_of = {int(i): k for k, i in enumerate(take)}
    for t1, t2, _, in1, in2 in loops:
        for t, pts in ((t1, in1), (t2, in2)):
            Pt = poses[at[t]].astype(np.float64); Po = Pn[node_of[at[t]]]
            for p in pts.astype(np.float64):
                pt.append(t)
                ps.append(np.float32(((Pt[:3, 0] * p[0] + Pt[:3, 1] * p[1]) + Pt[:3, 2] * p[2]) + Pt[:3, 3]))
                pd.append(((Po[:3, 0] * p[0] + Po[:3, 1] * p[1]) + Po[:3, 2] * p[2]) + Po[:3, 3])
    out = {}
    for kind, get in ((0, trk.get_processed_slice), (1, lambda i: trk.get_slice_mesh(i)[0])):
        recs = [get(i) for i in range(trk.num_slices())]
        ut = np.concatenate([np.full(len(r), trk.slice_info(i).utime, np.uint64) for i, r in enumerate(recs)])
        allr = np.concatenate(recs)
        xyz = np.stack([allr["x"], allr["y"], allr["z"]], 1); nrm = np.stack([allr["nx"], allr["ny"], allr["nz"]], 1)
        p, nn, rep, *_ = D.deform(times, poses[:, :3, 3], np.zeros(0, np.uint64), np.zeros((0, 3)), spacing, xyz, nrm, ut,
                                   points=(np.array(pt, np.uint64), np.array(ps, np.float32), np.array(pd, np.float64)))
        out[kind] = (p, nn, rep)
    return out


def _state(trk):
    n = trk.num_slices()
    return ([trk.get_deformed_slice(i).tobytes() for i in range(n)], [trk.get_deformed_slice_mesh(i).tobytes() for i in range(n)],
            [(t, p.tobytes()) for t, p, _ in trk.pose_graph_nodes()], trk.num_loops())


def test_tracker_loop_accept_reject_and_reset(built):
    import kintinuous_b200 as kb
    trk, _ = _track(kb)
    times, poses = _dense(trk)
    # 0.2 m / 0.025 rad off the trajectory: chi2 ~ 2 accepts it (the error spreads over 50 odometry factors), and the correction is
    # large enough that the deformation runs (|r_con| / constraints ~ 0.17, above its 0.1 early-out)
    C = _constraint(T1, T2, [0.01, -0.02, 0.01], [0.2, -0.1, 0.2])
    in1, in2 = _inliers(1, C)
    tracked_rel = np.linalg.inv(poses[T1].astype(np.float64)) @ poses[T2].astype(np.float64)
    rep = trk.close_loop(T1, T2, C, in1, in2, pose_spacing=0.0, node_spacing=0.05)
    print("accept:", rep.as_dict())
    take, Pn, orep, acc = P.close_loop(times, poses, [(T1, T2, C)], 0.0)
    assert rep.accepted == 1 and acc and trk.num_loops() == 1
    assert rep.iterations == orep["iterations"] and abs(rep.chi2_final - orep["chi2_final"]) <= 1e-6 * max(1.0, orep["chi2_final"])
    nodes = trk.pose_graph_nodes()
    assert [t for t, _, _ in nodes] == [int(times[i]) for i in take]
    Pd = np.array([p for _, p, _ in nodes], np.float64)
    dn = np.abs(Pd - Pn).max()
    assert dn <= 1e-5, dn                                                  # the nodes are float
    # the corrected relative pose (the tracker's own nodes) is closer to the constraint than the tracked one, rotation and translation
    rel = np.linalg.inv(Pd[T1]) @ Pd[T2]
    for sl in ((slice(0, 3), slice(0, 3)), (slice(0, 3), 3)):
        assert np.abs(rel - C)[sl].max() < 0.5 * np.abs(tracked_rel - C)[sl].max(), sl
    # the map: deformed for real, with kt_close_loop's node and inlier constraints, as pgo_oracle followed by deform_oracle.  This is a
    # parity check of the constraints and the hand-off, not of the deformation's quality: the synthetic trajectory is nearly a straight
    # line, rotation of the deformation nodes about it is held only by E_rot (whose Jacobian vanishes there at the identity), and the
    # reference's undamped Gauss-Newton (DeformationGraph.cpp:714-774) diverges on every correction large enough to pass its 0.1
    # early-out -- on the device and in the FP64 oracle alike, step for step.
    assert rep.map_deformed == 1 and rep.deform.deformed == 1 and rep.deform.iterations >= 1
    assert rep.deform.constraints == len(take) + 2 * len(in1)
    exp = _expected_map(trk, take, Pn, [(T1, T2, C, in1, in2)], 0.05)
    n = trk.num_slices()
    for kind, got in ((0, np.concatenate([trk.get_deformed_slice(i) for i in range(n)])),
                      (1, np.concatenate([trk.get_deformed_slice_mesh(i) for i in range(n)]))):
        p, nn, drep = exp[kind]
        g = np.stack([got["x"], got["y"], got["z"]], 1).astype(np.float64)
        orig = np.concatenate([trk.get_processed_slice(i) if kind == 0 else trk.get_slice_mesh(i)[0] for i in range(n)])
        moved = np.abs(g - np.stack([orig["x"], orig["y"], orig["z"]], 1)).max()
        print(f"kind {kind}: moved up to {moved:.3f} m, |map - oracle| {np.abs(g - p).max():.2e} m, deform {drep}")
        assert drep["deformed"] == 1 and drep["iterations"] == rep.deform.iterations
        assert abs(drep["constraint_error"] - rep.deform.constraint_error) <= 1e-5 * drep["constraint_error"]
        assert moved >= 0.05
        assert np.abs(g - p).max() <= 1e-5
    # a large perturbation: rejected, nothing changes
    before = _state(trk)
    Cbad = _constraint(T1, T2, [0.0, 0.3, 0.0], [0.5, 0.0, -0.4])
    _, _, brep, bacc = P.close_loop(times, poses, [(T1, T2, C), (T1, T2, Cbad)], 0.0)
    assert not bacc and brep["chi2_final"] > 100
    rep = trk.close_loop(T1, T2, Cbad, pose_spacing=0.0, node_spacing=0.05)
    print("reject:", rep.as_dict())
    assert rep.accepted == 0 and rep.map_deformed == 0 and rep.chi2_final > 100
    assert _state(trk) == before
    # pose_spacing > 0, a second loop on top of the first (consistent with the first loop's corrected trajectory)
    C2 = np.linalg.inv(Pn[50]) @ Pn[10] @ _constraint(0, 0, [0.001, 0.001, -0.002], [0.002, 0.003, -0.001])
    rep = trk.close_loop(50, 10, C2, pose_spacing=0.03, node_spacing=0.05)
    take2, Pn2, orep2, acc2 = P.close_loop(times, poses, [(T1, T2, C), (50, 10, C2)], 0.03)
    print("spacing:", rep.as_dict(), "oracle", orep2)
    assert rep.accepted == 1 and acc2 and trk.num_loops() == 2 and rep.nodes == len(take2) < len(times) and rep.map_deformed == 1
    assert np.abs(np.array([p for _, p, _ in trk.pose_graph_nodes()], np.float64) - Pn2).max() <= 1e-5
    # errors leave the state alone
    after = _state(trk)
    for bad in ((12345, T2, C), (T1, T1, C), (T1, T2, np.full((4, 4), np.nan)), (T1, T2, C * 1.01)):
        with pytest.raises(kb.KtError, match="error -1"):
            trk.close_loop(*bad, node_spacing=0.05)
    with pytest.raises(kb.KtError, match="error -3"):
        trk.close_loop(T1, T2, C, node_spacing=10.0)
    assert _state(trk) == after
    trk.reset()
    assert trk.num_loops() == 0 and trk.pose_graph_nodes() == []
    trk.close()


def test_close_loop_mid_sequence_does_not_touch_tracking(built):
    import kintinuous_b200 as kb
    _, ref = _track(kb)
    C = _constraint(30, 3, [0.002, 0.0, 0.001], [0.003, 0.0, 0.002])
    trk, mid = _track(kb, loop_at=35, loop_args=(30, 3, C, None, None, 0.0, 0.05))
    assert mid == ref
    assert trk.num_loops() == 1
    trk.close()


def test_tracker_refuses_a_65th_loop(built):
    import kintinuous_b200 as kb
    from kintinuous_b200 import synth
    trk = kb.Tracker(kb.Config.default(rows=ROWS, cols=COLS, vol=V, odometry=0, voxel_shift=2))
    for k in range(FRAMES):
        d, c = synth.render(k, COLS, ROWS)
        trk.process_frame(d, c, k)
    times, poses = _dense(trk)
    for i in range(64):                                                   # consistent loops: every one is accepted
        t1, t2 = 10 + i % 50, i % 10
        rep = trk.close_loop(t1, t2, np.linalg.inv(poses[t1].astype(np.float64)) @ poses[t2].astype(np.float64))
        assert rep.accepted == 1 and rep.loops == i + 1 and rep.map_deformed == 0, (i, rep.as_dict())
    before = [(t, p.tobytes()) for t, p, _ in trk.pose_graph_nodes()]
    with pytest.raises(kb.KtError, match="error -4"):
        trk.close_loop(59, 0, np.linalg.inv(poses[59].astype(np.float64)) @ poses[0].astype(np.float64))
    assert trk.num_loops() == 64 and [(t, p.tobytes()) for t, p, _ in trk.pose_graph_nodes()] == before
    trk.close()
