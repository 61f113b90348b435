"""The welded map mesh on the device: kt_op_mesh_volume_keyed against kt_op_mesh_volume and tests/weld_oracle.py, kt_op_weld_meshes
against weld_oracle.weld and against the union box's mesh, and the tracker's kt_get_slice_mesh_keys / kt_get_map_mesh /
kt_save_map_ply.  Everything is compared bit for bit: the weld only selects and copies records, and the keyed operator's records are
the plain operator's."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import map_oracle as M  # noqa: E402
from oracle import mesh_oracle as mo  # noqa: E402
from test_gpu_mesh import _dev, _random_volume, _store  # noqa: E402
from weld_oracle import keyed, weld  # noqa: E402

pytestmark = pytest.mark.gpu


def _sphere_volume(V, seed=1):
    z, y, x = np.meshgrid(*[np.arange(V)] * 3, indexing="ij")
    d = np.sqrt((x - 0.45 * V) ** 2 + (y - 0.52 * V) ** 2 + (z - 0.5 * V) ** 2) - 0.3 * V + 1.5 * np.sin(x * 0.4) * np.cos(y * 0.3)
    col = np.random.default_rng(seed).integers(0, 256, (V, V, V, 4), dtype=np.uint8)
    return mo.sdf_volume(d.astype(np.float32), color=col)


def test_keyed_operator_equals_the_operator_and_the_oracle(built):
    import kintinuous_b200 as kb
    table = mo.load_table()
    cases = [("random", *_random_volume(), 64, 0.9), ("sphere", *_sphere_volume(64), 64, 1.0)]
    for name, tl, cl, V, size in cases:
        for box, wrap, rw in (((0, V, 0, V, 0, V), (0, 0, 0), (0, 0, 0)), ((5, 40, 0, V, 9, V - 1), (13, V - 1, 7), (-7, 300, 2)),
                              ((V - 20, V, 3, V, 0, 30), (V + 5, 2 * V + 17, 3), (40, -2, -91))):
            ts, cs = _store(tl, cl, wrap)
            td, cd = _dev(ts, cs)
            v, t, e, k = kb.ops.mesh_volume_keyed(td, cd, V, [size] * 3, wrap, rw, box, 8)
            pv, pt = kb.ops.mesh_volume(td, cd, V, [size] * 3, wrap, rw, box, 8)
            assert v.tobytes() == pv.tobytes() and np.array_equal(t, pt), (name, box)
            _, _, own, cells = keyed(ts, cs, V, size, wrap, rw, box, 8, table)
            assert np.array_equal(e, own) and np.array_equal(k, cells), (name, box)
            assert len(t) > 100
    # capacity: the counts, nothing written
    import torch
    ts, cs = _store(*cases[1][1:3], (3, 4, 5))
    td, cd = _dev(ts, cs)
    st, nv, nt = kb.ops.mesh_volume_keyed_into(td, cd, 64, [1.0] * 3, (3, 4, 5), (0, 0, 0), (0, 64, 0, 64, 0, 64), 8, None, None, 0, None, None, 0)
    assert st == kb.binding.KT_ERR_CAPACITY and nv > 0 and nt > 0
    e = torch.full((nv * 4,), -7, dtype=torch.int32, device="cuda"); k = torch.full((nt * 4,), -7, dtype=torch.int32, device="cuda")
    v = torch.zeros(nv * 32, dtype=torch.uint8, device="cuda"); t = torch.zeros(nt * 3, dtype=torch.int32, device="cuda")
    st, _, _ = kb.ops.mesh_volume_keyed_into(td, cd, 64, [1.0] * 3, (3, 4, 5), (0, 0, 0), (0, 64, 0, 64, 0, 64), 8, v, e, nv, t, k, nt - 1)
    assert st == kb.binding.KT_ERR_CAPACITY and (e.cpu().numpy() == -7).all() and (k.cpu().numpy() == -7).all()


def _boxes(V, n, axis, rng):
    """n boxes tiling [0, V) along axis with random overlaps of 1 to 4 planes (the last ends at V - 1 on z, as a ZMinus slab)"""
    cuts = np.sort(rng.choice(np.arange(6, V - 6), n - 1, replace=False)) if n > 1 else np.array([], int)
    lo = np.concatenate([[0], cuts - rng.integers(1, 5, n - 1)]); hi = np.concatenate([cuts + 1, [V - 1 if axis == 2 else V]])
    out = []
    for a, b in zip(lo, hi):
        box = [0, V, 0, V, 0, V]; box[2 * axis] = int(a); box[2 * axis + 1] = int(b)
        out.append(tuple(box))
    return out


def test_weld_equals_the_oracle_and_the_union(built):
    import kintinuous_b200 as kb
    rng = np.random.default_rng(7)
    V, size = 64, 1.0
    vols = [_sphere_volume(V, 2), _random_volume(V, 5)]
    for trial in range(8):
        n = trial + 1
        axis = trial % 3
        tl, cl = vols[trial % 2]
        wrap = tuple(int(x) for x in rng.integers(0, 3 * V, 3)); rw = tuple(int(x) for x in rng.integers(-500, 500, 3))
        ts, cs = _store(tl, cl, wrap)
        td, cd = _dev(ts, cs)
        boxes = _boxes(V, n, axis, rng)
        order = list(rng.permutation(n))                                  # any box may be the later one
        meshes = [kb.ops.mesh_volume_keyed(td, cd, V, [size] * 3, wrap, rw, boxes[i], 8) for i in order]
        gv, gt, rep = kb.ops.weld_meshes(meshes)
        ov, ot, oe, oc, st = weld(meshes)
        assert gv.tobytes() == ov.tobytes() and np.array_equal(gt, ot), trial
        for key in ("output_verts", "output_tris", "repeated_cells", "dropped_triangles", "merged_vertices", "input_verts", "input_tris", "meshes"):
            assert rep[key] == st[key], (trial, key)
        union = (0, V, 0, V, 0, V - 1 if axis == 2 else V)
        uv, ut = kb.ops.mesh_volume(td, cd, V, [size] * 3, wrap, rw, union, 8)
        assert gv.tobytes() == uv.tobytes() and np.array_equal(gt, ut), trial
        again = kb.ops.weld_meshes(meshes)
        assert again[0].tobytes() == gv.tobytes() and again[1].tobytes() == gt.tobytes()
        if n > 1:
            assert rep["repeated_cells"] > 0
        print(f"weld of {n} boxes along axis {axis}: {rep['input_tris']} -> {rep['output_tris']} triangles, {rep['input_verts']} -> "
              f"{rep['output_verts']} vertices, {rep['repeated_cells']} repeated cells")


def test_weld_refusals_and_capacity(built):
    import torch
    import kintinuous_b200 as kb
    tl, cl = _sphere_volume(48)
    td, cd = _dev(tl, cl)
    meshes = [kb.ops.mesh_volume_keyed(td, cd, 48, [1.0] * 3, (0, 0, 0), (0, 0, 0), b, 8) for b in ((0, 30, 0, 48, 0, 48), (25, 48, 0, 48, 0, 48))]
    gv, gt, rep = kb.ops.weld_meshes(meshes)
    v = np.concatenate([m[0] for m in meshes]); t = np.concatenate([m[1] for m in meshes]).astype(np.uint32)
    e = np.concatenate([m[2] for m in meshes]).astype(np.int32); k = np.concatenate([m[3] for m in meshes]).astype(np.int32)
    vo = [0, len(meshes[0][0]), len(v)]; to = [0, len(meshes[0][1]), len(t)]
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()  # noqa: E731
    dv, dt, de, dk = dev(v), dev(t), dev(e), dev(k)
    nv, nt = len(gv), len(gt)
    for mv, mt in ((nv - 1, nt), (nv, nt - 1), (0, 0)):
        ob = torch.full(((nv + 4) * 32,), 0xAB, dtype=torch.uint8, device="cuda"); tb = torch.full(((nt + 4) * 12,), 0xCD, dtype=torch.uint8, device="cuda")
        st, cv, ct, _ = kb.ops.weld_meshes_into(dv, de, vo, dt, dk, to, ob, mv, tb, mt)
        assert st == kb.binding.KT_ERR_CAPACITY and (cv, ct) == (nv, nt)
        assert (ob.cpu().numpy() == 0xAB).all() and (tb.cpu().numpy() == 0xCD).all()
    ob = torch.zeros(nv * 32, dtype=torch.uint8, device="cuda"); tb = torch.zeros(nt * 12, dtype=torch.uint8, device="cuda")
    # n_meshes = 0, empty (null) offsets, an index outside its mesh, a bad axis, keys beyond 2^62
    lib = kb.load(); n1 = C.c_size_t(0); n2 = C.c_size_t(0)
    off0 = np.zeros(1, np.uint64)
    assert lib.kt_op_weld_meshes(C.c_void_p(dv.data_ptr()), C.c_void_p(de.data_ptr()), off0.ctypes.data_as(C.c_void_p), C.c_void_p(dt.data_ptr()),
                                 C.c_void_p(dk.data_ptr()), off0.ctypes.data_as(C.c_void_p), 0, C.c_void_p(ob.data_ptr()), C.c_size_t(nv),
                                 C.c_void_p(tb.data_ptr()), C.c_size_t(nt), C.byref(n1), C.byref(n2), None, None) == -1
    assert lib.kt_op_weld_meshes(C.c_void_p(dv.data_ptr()), C.c_void_p(de.data_ptr()), None, C.c_void_p(dt.data_ptr()), C.c_void_p(dk.data_ptr()),
                                 None, 2, C.c_void_p(ob.data_ptr()), C.c_size_t(nv), C.c_void_p(tb.data_ptr()), C.c_size_t(nt),
                                 C.byref(n1), C.byref(n2), None, None) == -1
    bad_t = t.copy(); bad_t[-1, 2] = len(meshes[1][0])                    # one past the second mesh's vertices
    with pytest.raises(kb.KtError, match="error -1.*outside"):
        kb.ops.weld_meshes_into(dv, de, vo, dev(bad_t), dk, to, ob, nv, tb, nt)
    bad_e = e.copy(); bad_e[3, 3] = 3
    with pytest.raises(kb.KtError, match="error -1.*axis"):
        kb.ops.weld_meshes_into(dv, dev(bad_e), vo, dt, dk, to, ob, nv, tb, nt)
    far = e.copy(); far[0, :3] = -2 ** 30; far[1, :3] = 2 ** 30
    with pytest.raises(kb.KtError, match="error -1.*2\\^62"):
        kb.ops.weld_meshes_into(dv, dev(far), vo, dt, dk, to, ob, nv, tb, nt)
    # no triangles: nothing out
    st, cv, ct, _ = kb.ops.weld_meshes_into(None, None, [0, 0], None, None, [0, 0], ob, nv, tb, nt)
    assert (st, cv, ct) == (0, 0, 0)
    # a valid call after the refusals still works
    again = kb.ops.weld_meshes(meshes)
    assert again[0].tobytes() == gv.tobytes() and np.array_equal(again[1], gt)


# ---- the tracker ------------------------------------------------------------------------------------------------------------
ROWS, COLS, V, FRAMES = 240, 320, 256, 60


def _track(kb, meshing=True, act=None):
    from kintinuous_b200 import synth
    trk = kb.Tracker(kb.Config.default(rows=ROWS, cols=COLS, vol=V, odometry=0, voxel_shift=2))
    if meshing:
        trk.set_slice_meshing(True, 8)
    poses, launches, shifted = [], [], []
    for k in range(FRAMES):
        if act is not None and k == FRAMES // 2:
            act(trk)
        d, c = synth.render(k, COLS, ROWS)
        l0 = trk.launch_count()
        p = trk.process_frame(d, c, k)
        launches.append(trk.launch_count() - l0); shifted.append(sum(a != b for a, b in zip(p.voxel_wrap, poses[-1][1])) if poses else 0)
        poses.append((bytes(p), tuple(p.voxel_wrap)))
    trk.finalise()
    return trk, [p for p, _ in poses], launches, shifted


def _slices(trk):
    n = trk.num_slices()
    return [trk.get_slice_mesh(i) + trk.get_slice_mesh_keys(i) for i in range(n)]


def test_tracker_map_mesh(built, tmp_path):
    import kintinuous_b200 as kb
    off, off_poses, off_launches, shifted = _track(kb, meshing=False)
    with pytest.raises(kb.KtError, match="error -3"):
        off.map_mesh(0)                                                   # no slice mesh
    with pytest.raises(kb.KtError, match="error -3"):
        off.get_slice_mesh_keys(0)
    off.close()
    ref, ref_poses, ref_launches, _ = _track(kb)
    mid = {}

    def act(trk):
        with pytest.raises(kb.KtError, match="error -3"):
            trk.map_mesh(1)                                               # never deformed
        mid["mesh"] = trk.map_mesh(0, True)
        trk.save_map_ply(str(tmp_path / "mid.ply"), 0, True)
        dp = [trk.dense_pose(i) for i in range(trk.num_dense_poses())]
        from test_gpu_map import _rigid
        trk.deform_map([(t, _rigid(p)) for t, p, _ in dp], node_spacing=0.05)
        mid["covered"] = trk.num_slices()
        mid["last"] = (dp[-1][1], np.asarray(_rigid(dp[-1][1]), np.float32))
    trk, poses, launches, _ = _track(kb, act=act)
    # the export between frames changes no pose, no slice mesh and no key; meshing adds exactly the mesh's three launches per shifted axis
    assert poses == ref_poses == off_poses
    rs, ts = _slices(ref), _slices(trk)
    assert len(rs) == len(ts) >= 4
    for a, b in zip(rs, ts):
        assert a[0].tobytes() == b[0].tobytes() and all(np.array_equal(x, y) for x, y in zip(a[1:], b[1:]))
    assert any(shifted)
    for k in range(1, FRAMES):                  # a mesh is one count launch, and a vertex and a triangle launch when it has vertices
        assert ref_launches[k] == off_launches[k] if not shifted[k] else off_launches[k] < ref_launches[k] <= off_launches[k] + 3 * shifted[k], k

    # which 0, weld 1: the oracle weld of the recorded slice meshes and keys
    gv, gt, rep = ref.map_mesh(0, True)
    print("welded:", rep)
    ov, ot, oe, oc, st = weld(rs)
    assert gv.tobytes() == ov.tobytes() and np.array_equal(gt, ot)
    # no edge twice; each output cell's triangles are exactly those of the latest slice that meshed it
    assert len(np.unique(oe, axis=0)) == len(oe)
    latest = {}
    for i, s in enumerate(rs):
        for c in map(tuple, s[3][:, :3]):
            latest.setdefault(c, {}); latest[c][i] = latest[c].get(i, 0) + 1
    cells, counts = np.unique(oc[:, :3], axis=0, return_counts=True)
    assert all(latest[tuple(c)][max(latest[tuple(c)])] == k for c, k in zip(cells, counts))
    # On this stream no cell is meshed by two slices: an x shift clears round_up16(|n|) planes, the overlap among them (Q13), and the y / z
    # slabs that leave lie behind the camera, where nothing was observed.  Repeated cells are covered by the operator tests above.
    assert rep["repeated_cells"] == st["repeated_cells"] and rep["merged_vertices"] == st["merged_vertices"]
    assert (rep["meshes"], rep["moved_meshes"], rep["input_tris"]) == (len(rs), 0, sum(len(s[1]) for s in rs))
    assert rep["output_verts"] == len(gv) and rep["output_tris"] == len(gt) == rep["input_tris"] - rep["dropped_triangles"]
    # weld 0: kt_save_mesh_ply's content, and its bytes
    cv, ct, crep = ref.map_mesh(0, False)
    offs = np.cumsum([0] + [len(s[0]) for s in rs[:-1]])
    assert cv.tobytes() == np.concatenate([s[0] for s in rs]).tobytes()
    assert np.array_equal(ct, np.concatenate([s[1].astype(np.int64) + o for s, o in zip(rs, offs)]))
    ref.save_mesh_ply(str(tmp_path / "a.ply")); ref.save_map_ply(str(tmp_path / "b.ply"), 0, False)
    assert (tmp_path / "a.ply").read_bytes() == (tmp_path / "b.ply").read_bytes()
    ref.save_map_ply(str(tmp_path / "w.ply"), 0, True)
    blob = (tmp_path / "w.ply").read_bytes()
    assert f"element vertex {len(gv)}\n".encode() in blob and f"element face {len(gt)}\n".encode() in blob
    with pytest.raises(kb.KtError, match="error -1"):
        ref.map_mesh(2)

    # which 1 after a deformation: the same triangles, vertices deformed (covered slices) or moved rigidly (later ones)
    covered = mid["covered"]; n = len(ts)
    assert 1 <= covered < n
    g0v, g0t, _ = trk.map_mesh(0, True)
    g1v, g1t, rep1 = trk.map_mesh(1, True)
    print("welded, corrected:", rep1)
    assert np.array_equal(g1t, g0t) and rep1["moved_meshes"] == n - covered
    Rc, tc = M.correction(*mid["last"])
    moved = [trk.get_deformed_slice_mesh(i) for i in range(covered)] + [M.rigid_move(ts[i][0], Rc, tc) for i in range(covered, n)]
    want = weld([(moved[i],) + tuple(ts[i][1:]) for i in range(n)])
    assert g1v.tobytes() == want[0].tobytes()
    c1v, c1t, _ = trk.map_mesh(1, False)
    assert c1v.tobytes() == np.concatenate(moved).tobytes() and np.array_equal(c1t, np.concatenate([s[1].astype(np.int64) + o for s, o in zip(ts, np.cumsum([0] + [len(s[0]) for s in ts[:-1]]))]))

    # a reset clears the slices and the correction
    trk.reset()
    with pytest.raises(kb.KtError, match="error -3"):
        trk.map_mesh(0)
    with pytest.raises(kb.KtError, match="error -3"):
        trk.map_mesh(1)
    ref.close(); trk.close()
