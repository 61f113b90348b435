"""The whole-map export on the GPU: kt_op_voxel_grid (kt_map.cu) bit-identical to the float32 restatement in oracle/map_oracle.py, and
kt_get_map_cloud / kt_save_map_pcd on the tracker: the recorded map, its overlap filter, the corrected map after a deformation, the
.pcd file, and no effect on tracking.  "Bit-identical" lets two NaNs match whatever their payloads (map_oracle.same_bits)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from conftest import ROOT

sys.path.insert(0, ROOT)
from oracle import map_oracle as M  # noqa: E402

pytestmark = pytest.mark.gpu

LEAF = np.float32(6.0 / 512)


def _dtype(kind):
    from kintinuous_b200.binding import POINT_DTYPE, POINT_NORMAL_DTYPE
    return POINT_DTYPE if kind == 0 else POINT_NORMAL_DTYPE


def _fill(rng, p):
    for c in ("r", "g", "b", "a"):
        p[c] = rng.integers(0, 256, len(p))
    if "nx" in p.dtype.names:
        nrm = rng.normal(size=(len(p), 3)).astype(np.float32)
        p["nx"], p["ny"], p["nz"] = nrm.T
        p["curvature"] = rng.uniform(0, 0.3, len(p)).astype(np.float32)
        p["_p0"] = 1.0
    return p


def _run(pts, kind, leaf, capacity=None):
    import torch
    import kintinuous_b200 as kb
    cap = len(pts) if capacity is None else capacity
    d = torch.from_numpy(np.ascontiguousarray(pts).view(np.uint8).copy()).cuda() if len(pts) else None
    out = torch.full((max(cap, 1) * pts.dtype.itemsize,), 0xAB, dtype=torch.uint8, device="cuda")
    n, skip = kb.ops.voxel_grid(d, len(pts), kind, float(leaf), out, cap)
    return out.cpu().numpy().view(pts.dtype)[:min(n, cap)].copy(), n, skip


def _check(pts, kind, leaf, label):
    want, wskip = M.voxel_grid(pts, leaf)
    got, n, skip = _run(pts, kind, leaf)
    assert n == len(want) and skip == int(wskip), (label, n, len(want), skip, wskip)
    assert M.same_bits(got, want), label
    return got, want


def _leafy(rng, kind, n_leaves, lo=-3.0, leaf=LEAF, max_per_leaf=30):
    """Points in n_leaves distinct leaves of a 600^3 grid starting at lo, 1 .. max_per_leaf per leaf, shuffled."""
    cells = rng.choice(600 ** 3, n_leaves, replace=False)
    ijk = np.stack([cells % 600, (cells // 600) % 600, cells // 360000], -1)
    cnt = rng.integers(1, max_per_leaf + 1, n_leaves)
    ijk = np.repeat(ijk, cnt, axis=0)
    xyz = ((ijk + rng.uniform(0.02, 0.98, ijk.shape)) * float(leaf) + lo).astype(np.float32)
    p = np.zeros(len(xyz), _dtype(kind))
    p["x"], p["y"], p["z"] = xyz.T
    return _fill(rng, p)[rng.permutation(len(p))]


@pytest.mark.parametrize("kind", [0, 1])
def test_operator_is_bit_identical_to_the_oracle(built, kind):
    rng = np.random.default_rng(10 + kind)
    # 10^6 points, 1 - 30 per leaf, negative and positive coordinates
    pts = _leafy(rng, kind, 64_500)
    assert 900_000 < len(pts) < 1_100_000 and pts["x"].min() < 0
    got, want = _check(pts, kind, LEAF, "random")
    again, _, _ = _run(pts, kind, LEAF)
    assert again.tobytes() == got.tobytes()                                              # deterministic, byte for byte
    # points exactly on leaf boundaries: a power-of-two leaf (exact products) and the voxel edge (products rounded either way)
    k = rng.integers(-200, 200, (20000, 3)).astype(np.float32)
    for leaf, xyz in ((np.float32(0.25), k * np.float32(0.25)), (LEAF, k * LEAF)):
        p = _fill(rng, np.zeros(len(xyz), _dtype(kind)))
        p["x"], p["y"], p["z"] = xyz.T
        _check(p, kind, leaf, f"boundaries {leaf}")
    # -0.0 and +0.0, alone and together in a leaf
    p = _fill(rng, np.zeros(6, _dtype(kind)))
    p["x"] = [-0.0, 0.0, -0.0, 0.3, 0.3, -0.0]; p["y"] = [0.0, 0.0, 0.5, 0.5, -0.0, 1.0]; p["z"] = [1.0, 1.0, 1.0, 1.0, 1.0, -0.0]
    got, _ = _check(p, kind, np.float32(0.1), "signed zeros")
    assert np.signbit(got["z"]).any()
    # one leaf holding 10^5 points
    p = _fill(rng, np.zeros(100_000, _dtype(kind)))
    # leaf 171 of x spans [2.0039, 2.0156) m, leaf -86 of y [-1.0078, -0.9961) m, leaf 42 of z [0.4922, 0.5039) m
    p["x"] = rng.uniform(2.005, 2.015, len(p)).astype(np.float32); p["y"] = rng.uniform(-1.007, -0.997, len(p)).astype(np.float32); p["z"] = 0.5
    got, _ = _check(p, kind, LEAF, "one big leaf")
    assert len(got) == 1
    # more than INT_MAX cells (100 m x 100 m x 3 m at the voxel edge): filtered on 64-bit keys, PCL would have skipped
    p = _fill(rng, np.zeros(200_000, _dtype(kind)))
    p["x"] = rng.uniform(-50, 50, len(p)).astype(np.float32); p["y"] = rng.uniform(-50, 50, len(p)).astype(np.float32)
    p["z"] = rng.uniform(0, 3, len(p)).astype(np.float32)
    p = np.concatenate([p, p[:5000]])                                                      # some leaves with two points
    got, want = _check(p, kind, LEAF, "beyond INT_MAX")
    assert M.grid(p, LEAF)[3] and len(got) < len(p)
    # n = 0 and n = 1
    got, n, skip = _run(p[:0], kind, LEAF)
    assert (n, skip, len(got)) == (0, 0, 0)
    _check(p[:1], kind, LEAF, "one point")


def test_operator_nan_normals_capacity_and_errors(built):
    import kintinuous_b200 as kb
    rng = np.random.default_rng(3)
    pts = _leafy(rng, 1, 5000)
    pts["nx"][::7] = np.nan; pts["curvature"][::11] = np.nan
    got, want = _check(pts, 1, LEAF, "nan normals")
    assert np.isnan(got["nx"]).any() and not np.isnan(got["x"]).any()
    # a capacity below the output still returns the full count, and the first records
    small, n, _ = _run(pts, 1, LEAF, capacity=100)
    assert n == len(want) and len(small) == 100 and M.same_bits(small, want[:100])
    small, n, _ = _run(pts, 1, LEAF, capacity=0)
    assert n == len(want)
    # a non-finite position is refused
    for bad in (np.nan, np.inf):
        p = pts.copy(); p["y"][17] = bad
        with pytest.raises(kb.KtError, match="error -1.*non-finite"):
            _run(p, 1, LEAF)
    with pytest.raises(kb.KtError, match="error -1"):
        _run(pts, 2, LEAF)
    with pytest.raises(kb.KtError, match="error -1"):
        _run(pts, 1, np.float32(0.0))


# ---- the tracker ------------------------------------------------------------------------------------------------------------
ROWS, COLS, V, FRAMES = 240, 320, 256, 60


def _track(kb, act=None, n=FRAMES):
    from kintinuous_b200 import synth
    trk = kb.Tracker(kb.Config.default(rows=ROWS, cols=COLS, vol=V, odometry=0, voxel_shift=2))
    trk.set_slice_processing(True, 8)
    poses, traces = [], []
    for k in range(n):
        if act is not None and k == n // 2:
            act(trk)
        d, c = synth.render(k, COLS, ROWS)
        poses.append(bytes(trk.process_frame(d, c, k)))
        traces.append(trk.trace().tobytes())
    trk.finalise()
    return trk, poses, traces


def _rigid(p):
    from scipy.spatial.transform import Rotation
    R = Rotation.from_rotvec([0.05, 0.25, -0.04]).as_matrix(); T = np.array([0.4, -0.25, 0.5])
    q = np.eye(4); q[:3, :3] = R @ p[:3, :3]; q[:3, 3] = R @ p[:3, 3] + T
    return q


def test_tracker_map_export(built, tmp_path):
    import kintinuous_b200 as kb
    ref, ref_poses, ref_traces = _track(kb)
    mid = {}

    def act(trk):
        # mid-run: the corrected map does not exist yet; export both recorded maps and a file, then deform rigidly
        with pytest.raises(kb.KtError, match="error -3"):
            trk.map_cloud(1)
        mid["cloud"] = trk.map_cloud(0, True)[0]
        trk.save_map_pcd(str(tmp_path / "mid.pcd"), 0, True)
        dp = [trk.dense_pose(i) for i in range(trk.num_dense_poses())]
        trk.deform_map([(t, _rigid(p)) for t, p, _ in dp], node_spacing=0.05)
        mid["covered"] = trk.num_slices()
        mid["last"] = (dp[-1][1], np.asarray(_rigid(dp[-1][1]), np.float32))
    trk, poses, traces = _track(kb, act)
    # exporting and deforming mid-run changes no pose and no trace
    assert poses == ref_poses and traces == ref_traces
    assert M.read_pcd((tmp_path / "mid.pcd").read_bytes(), mid["cloud"].dtype).tobytes() == mid["cloud"].tobytes()

    # the recorded map: the concatenation of the processed slices, then the voxel grid over it
    n = ref.num_slices()
    slices = [ref.get_processed_slice(i) for i in range(n)]
    cat = np.concatenate(slices)
    cloud, rep = ref.map_cloud(0, False)
    print("recorded:", rep)
    assert cloud.tobytes() == cat.tobytes()
    assert (rep["input_points"], rep["output_points"], rep["slices"], rep["moved_slices"]) == (len(cat), len(cat), n, 0)
    dd, rep = ref.map_cloud(0, True)
    print("recorded, dedupe:", rep)
    want, skip = M.voxel_grid(cat, np.float32(ref.voxel_size))
    assert M.same_bits(dd, want) and rep["pcl_would_skip"] == int(skip) == 0
    assert len(dd) <= len(cat) and rep["output_points"] == len(dd) and rep["input_points"] == len(cat)
    # the files parse back to the same clouds, in PCL's layout
    for dedupe, c in ((False, cloud), (True, dd)):
        path = tmp_path / f"map{int(dedupe)}.pcd"
        ref.save_map_pcd(str(path), 0, dedupe)
        blob = path.read_bytes()
        assert blob == M.pcd_bytes(c)
        assert M.read_pcd(blob, c.dtype).tobytes() == c.tobytes()
    # a capacity of one point returns the full count and the first point
    buf = np.zeros(1, cloud.dtype); cnt = C.c_size_t(0)
    assert ref.lib.kt_get_map_cloud(ref.h, 0, 0, buf.ctypes.data_as(C.c_void_p), C.c_size_t(1), C.byref(cnt), None) == 0
    assert cnt.value == len(cat) and buf.tobytes() == cat[:1].tobytes()
    with pytest.raises(kb.KtError, match="error -1"):
        ref.map_cloud(2)
    with pytest.raises(kb.KtError, match="error -3"):
        ref.map_cloud(1)                                                                  # never deformed

    # the corrected map: deformed copies of the covered slices, the rest moved by the last correction
    covered = mid["covered"]
    n = trk.num_slices()
    assert 1 <= covered < n
    got, rep = trk.map_cloud(1, False)
    print("corrected:", rep)
    head = np.concatenate([trk.get_deformed_slice(i) for i in range(covered)])
    tail_in = np.concatenate([trk.get_processed_slice(i) for i in range(covered, n)])
    assert (rep["slices"], rep["moved_slices"], rep["input_points"]) == (n, n - covered, len(head) + len(tail_in))
    assert got[:len(head)].tobytes() == head.tobytes()
    Rc, tc = M.correction(*mid["last"])
    tail = M.rigid_move(tail_in, Rc, tc)
    g = got[len(head):]
    for f in ("x", "y", "z", "nx", "ny", "nz"):
        assert np.abs(g[f].astype(np.float64) - tail[f]).max() <= 1e-6, f
    # against the correction in FP64: the pose's rigid move, as the caller stated it
    Rr = _rigid(np.eye(4))
    xyz = np.stack([tail_in[c] for c in "xyz"], -1).astype(np.float64) @ Rr[:3, :3].T + Rr[:3, 3]
    dev = np.abs(np.stack([g[c] for c in "xyz"], -1) - xyz).max()
    print(f"moved slices vs the FP64 rigid move: {dev:.2e} m")
    assert dev <= 1e-5
    for f in ("r", "g", "b", "a", "curvature", "_p0", "_p1"):
        assert np.array_equal(g[f], tail_in[f]), f
    dd, rep = trk.map_cloud(1, True)
    want, _ = M.voxel_grid(got, np.float32(trk.voxel_size))
    assert M.same_bits(dd, want) and len(dd) <= len(got)
    path = tmp_path / "map_opt.pcd"
    trk.save_map_pcd(str(path), 1, False)
    assert M.read_pcd(path.read_bytes(), got.dtype).tobytes() == got.tobytes()

    # a reset clears the correction: new slices, no corrected map
    from kintinuous_b200 import synth
    trk.reset()
    for k in range(8):
        d, c = synth.render(k, COLS, ROWS)
        trk.process_frame(d, c, k)
    trk.finalise()
    assert trk.map_cloud(0)[1]["slices"] >= 1
    with pytest.raises(kb.KtError, match="error -3"):
        trk.map_cloud(1)
    trk.close(); ref.close()


def test_tracker_without_processed_slices(built):
    import kintinuous_b200 as kb
    from kintinuous_b200 import synth
    trk = kb.Tracker(kb.Config.default(rows=ROWS, cols=COLS, vol=V, odometry=0, voxel_shift=2))
    for k in range(4):
        d, c = synth.render(k, COLS, ROWS)
        trk.process_frame(d, c, k)
    trk.finalise()
    with pytest.raises(kb.KtError, match="error -3"):
        trk.map_cloud(0)
    with pytest.raises(kb.KtError, match="error -3"):
        trk.save_map_pcd(os.devnull, 0, True)
    trk.close()


def test_overlap_planes_merge(built):
    """640 x 480 into 512^3, 300 frames with a shift every 2 voxels: neighbouring slices repeat their overlap planes, and the map's voxel
    grid merges them into one point per leaf, bit-identical to the oracle."""
    import kintinuous_b200 as kb
    from kintinuous_b200 import synth
    trk = kb.Tracker(kb.Config.default(rows=480, cols=640, vol=512, odometry=0, voxel_shift=2))
    trk.set_slice_processing(True, 8)
    for k in range(300):
        d, c = synth.render(k, 640, 480)
        trk.process_frame(d, c, k)
    trk.finalise()
    n = trk.num_slices()
    slices = [trk.get_processed_slice(i) for i in range(n)]
    cat = np.concatenate(slices)
    dd, rep = trk.map_cloud(0, True)
    want, _ = M.voxel_grid(cat, np.float32(trk.voxel_size))
    assert M.same_bits(dd, want) and rep["input_points"] == len(cat)
    keys = M.leaf_keys(cat, np.float32(trk.voxel_size))
    sid = np.repeat(np.arange(n), [len(s) for s in slices])
    o = np.lexsort((sid, keys))
    k, sd = keys[o], sid[o]
    first = np.ones(len(k), bool); first[1:] = k[1:] != k[:-1]
    multi = np.unique(k[~first & (sd != np.roll(sd, 1))])
    print(f"{n} slices, {len(cat)} points, {len(dd)} leaves, {len(multi)} of them held points of more than one slice")
    assert len(multi) > 0 and len(dd) < len(cat)
    trk.close()
