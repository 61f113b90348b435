"""kt_mesh.cu (marching cubes over a box of the cyclic TSDF) through the C ABI: kt_op_mesh_volume against the numpy restatement
oracle/mesh_oracle.py, against kt_op_extract_slice, and the tracker's slice meshes (kt_set_slice_meshing, kt_get_slice_mesh,
kt_get_live_mesh, kt_save_mesh_ply).

Tolerances: triangle index arrays, colours and alpha identical; positions <= 1e-6 m (the oracle repeats interp's float32 order but not
its fused multiply-add nor the approximate reciprocal); normals <= 1e-5 (float32 gradient blend against float64).  Everything else
(determinism, wrap invariance, tracker slices against the operator) is bit for bit."""
import os
import sys

import numpy as np
import pytest

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import mesh_oracle as mo  # noqa: E402
from test_mesh_table import analytic_volume  # noqa: E402

pytestmark = pytest.mark.gpu


def _store(tsdf_l, col_l, wrap):
    """logical -> storage order at `wrap` (logical x is stored at (x + wrap.x) mod V)"""
    V = tsdf_l.shape[0]
    w = [int(v) % V for v in wrap]
    return np.roll(tsdf_l, (w[2], w[1], w[0]), (0, 1, 2)), np.roll(col_l, (w[2], w[1], w[0]), (0, 1, 2))


def _dev(t, c):
    import torch
    return torch.from_numpy(np.ascontiguousarray(t)).cuda(), torch.from_numpy(np.ascontiguousarray(c)).cuda()


def _mesh(kb, t, c, V, size, wrap, rw, box, cull=8):
    td, cd = _dev(t, c)
    return kb.ops.mesh_volume(td, cd, V, [size] * 3, wrap, rw, box, cull)


def _compare(got, want, label):
    gv, gt = got; wv, wt = want
    assert len(gv) == len(wv) and gt.shape == wt.shape, (label, len(gv), len(wv), gt.shape, wt.shape)
    assert np.array_equal(gt, wt), label
    for ch in ("r", "g", "b", "a", "_pad"):
        assert np.array_equal(gv[ch], wv[ch]), (label, ch)
    dp = max(float(np.abs(gv[k].astype(np.float64) - wv[k]).max()) for k in ("x", "y", "z")) if len(gv) else 0.0
    dn = max(float(np.abs(gv[k].astype(np.float64) - wv[k]).max()) for k in ("nx", "ny", "nz")) if len(gv) else 0.0
    print(f"{label}: {len(gv)} vertices, {len(gt)} triangles; max |dpos| {dp:.2e} m, max |dnormal| {dn:.2e}")
    assert dp <= 1e-6 and dn <= 1e-5, (label, dp, dn)


def _random_volume(V=64, seed=3):
    rng = np.random.default_rng(seed)
    # smooth-ish field plus noise so that most cells are near the surface, with the special values 0 and 32767 mixed in
    z, y, x = np.meshgrid(np.arange(V), np.arange(V), np.arange(V), indexing="ij")
    f = np.sin(x / 5.0) * np.cos(y / 7.0) + np.sin(z / 6.0) * 0.7 + rng.normal(0, 0.35, (V, V, V))
    t = np.clip(f * 20000, -32767, 32767).astype(np.int16)
    t[rng.random((V, V, V)) < 0.01] = 0
    t[rng.random((V, V, V)) < 0.01] = 32767
    c = rng.integers(0, 256, (V, V, V, 4), dtype=np.uint8)
    c[..., 3] = rng.integers(0, 40, (V, V, V))                     # weights below the cull and 0 (never observed) included
    return t, c


BOXES_FULL = lambda V: (0, V, 0, V, 0, V)  # noqa: E731


def test_kernel_matches_oracle(built):
    """The analytic volumes at 128, the random one at 64 and at 96 (not a power of two: cyclic reduction by subtraction); the third wrap
    is beyond one volume length on every axis."""
    import kintinuous_b200 as kb
    table = mo.load_table()
    cases = []
    for name in ("sphere", "torus", "two_spheres"):
        t, c = analytic_volume(name)
        cases.append((name, t, c, 128, 1.28))
    for V in (64, 96):
        t, c = _random_volume(V)
        cases.append((f"random{V}", t, c, V, 0.9))
    for name, tl, cl, V, size in cases:
        boxes = [BOXES_FULL(V), (5, V // 2 + 3, 0, V, V // 4 + 1, V - 3), (V - 20, V, 3, V, 0, 30)]
        wraps = [(0, 0, 0), (13, V - 1, 7), (V + 5, 2 * V + 17, 3 * V - 1)]
        for bi, box in enumerate(boxes):
            for wi, wrap in enumerate(wraps):
                if bi and wi == 1:
                    continue
                ts, cs = _store(tl, cl, wrap)
                rw = (wi * 3 - 2, -wi, 5 * wi)
                for cull in ((8, 0) if name.startswith("random") else (8,)):
                    got = _mesh(kb, ts, cs, V, size, wrap, rw, box, cull)
                    want = mo.mesh(ts, cs, V, size, wrap, rw, box, cull, table)
                    _compare(got, want, f"{name} box{bi} wrap{wi} cull{cull}")
                    if bi == 0 and not name.startswith("random"):
                        assert len(got[0]) > 1000


def test_vertices_are_extracted_points(built):
    """Every vertex whose edge has two non-zero ends is, bit for bit, one of extract_slice's points on the same volume (box extended by
    one plane on each upper side)."""
    import torch
    import kintinuous_b200 as kb
    from kintinuous_b200.binding import POINT_DTYPE
    for name, (tl, cl), V, size in (("torus", analytic_volume("torus"), 128, 1.28), ("random", _random_volume(), 64, 0.9)):
        wrap, rw = (V + 9, 3, V - 2), (4, -7, 1)
        ts, cs = _store(tl, cl, wrap)
        box = (3, V - 10, 0, V // 2, 7, V)
        verts, _ = _mesh(kb, ts, cs, V, size, wrap, rw, box, 8)
        td, cd = _dev(ts, cs)
        cap = 3 * V ** 3
        out = torch.zeros(cap * 32, dtype=torch.uint8, device="cuda")
        ebox = (box[0], min(box[1] + 1, V), box[2], min(box[3] + 1, V), box[4], min(box[5] + 1, V))
        n = kb.ops.extract_slice(td, [size] * 3, V, out, cap, wrap, cd, ebox, 1, rw)
        pts = out[:n * 32].cpu().numpy().view(POINT_DTYPE)
        ext = set(map(bytes, np.stack([pts["x"], pts["y"], pts["z"]], -1).astype("<f4")))
        # which vertices have two non-zero ends: the oracle knows each vertex's edge
        _, _, owners = mo.mesh(ts, cs, V, size, wrap, rw, box, 8, return_owners=True)
        T = mo.logical(ts, wrap, V).astype(np.int32)
        x, y, z, a = owners.T
        d = np.zeros((len(a), 3), np.int64); d[np.arange(len(a)), a] = 1
        nz = (T[z, y, x] != 0) & (T[z + d[:, 2], y + d[:, 1], x + d[:, 0]] != 0)
        vx = np.stack([verts["x"], verts["y"], verts["z"]], -1).astype("<f4")
        hits = np.array([bytes(r) in ext for r in vx])
        print(f"{name}: {int(nz.sum())} of {len(verts)} vertices have two non-zero ends; all in the {n} extracted points: {bool(hits[nz].all())}")
        assert nz.sum() > 1000 and hits[nz].all()


def test_wrap_invariance_determinism_capacity(built):
    import torch
    import kintinuous_b200 as kb
    tl, cl = _random_volume(V=48, seed=11)
    V, size, box = 48, 0.7, (2, 40, 0, 48, 5, 48)
    rw = (3, -4, 9)
    ref = None
    for wrap in ((0, 0, 0), (17, 31, 47), (100, 5, 96 + 13)):
        ts, cs = _store(tl, cl, wrap)
        got = _mesh(kb, ts, cs, V, size, wrap, rw, box)
        again = _mesh(kb, ts, cs, V, size, wrap, rw, box)
        assert got[0].tobytes() == again[0].tobytes() and np.array_equal(got[1], again[1])
        if ref is None:
            ref = got
        assert got[0].tobytes() == ref[0].tobytes() and np.array_equal(got[1], ref[1]), wrap
    # positions move only through real_voxel_wrap
    ts, cs = _store(tl, cl, (0, 0, 0))
    shifted = _mesh(kb, ts, cs, V, size, (0, 0, 0), (rw[0] + 2, rw[1], rw[2] - 1), box)
    cell = np.float32(size) / np.float32(V)
    assert np.abs(shifted[0]["x"] - ref[0]["x"] - 2 * cell).max() < 1e-6 and np.abs(shifted[0]["z"] - ref[0]["z"] + cell).max() < 1e-6
    assert np.array_equal(shifted[0]["y"], ref[0]["y"]) and np.array_equal(shifted[1], ref[1])
    # capacity: counts returned, nothing written
    nv, nt = len(ref[0]), len(ref[1])
    td, cd = _dev(ts, cs)
    for mv, mt in ((nv - 1, nt), (nv, nt - 1), (0, 0)):
        vb = torch.full(((nv + 8) * 32,), 0xAB, dtype=torch.uint8, device="cuda")
        tb = torch.full(((nt + 8) * 12,), 0xCD, dtype=torch.uint8, device="cuda")
        st, gv, gt = kb.ops.mesh_volume_into(td, cd, V, [size] * 3, (0, 0, 0), rw, box, 8, vb, mv, tb, mt)
        assert st == kb.binding.KT_ERR_CAPACITY and (gv, gt) == (nv, nt)
        assert (vb.cpu().numpy() == 0xAB).all() and (tb.cpu().numpy() == 0xCD).all()
    vb = torch.full(((nv + 8) * 32,), 0xAB, dtype=torch.uint8, device="cuda")
    tb = torch.full(((nt + 8) * 12,), 0xCD, dtype=torch.uint8, device="cuda")
    st, gv, gt = kb.ops.mesh_volume_into(td, cd, V, [size] * 3, (0, 0, 0), rw, box, 8, vb, nv, tb, nt)
    assert st == 0 and (gv, gt) == (nv, nt)
    assert (vb.cpu().numpy()[nv * 32:] == 0xAB).all() and (tb.cpu().numpy()[nt * 12:] == 0xCD).all()
    assert vb.cpu().numpy()[:nv * 32].tobytes() == ref[0].tobytes()


def _canon(p):
    a = np.ascontiguousarray(p).view(np.uint64).reshape(len(p), 4)
    return a[np.lexsort(a.T[::-1])] if len(a) else a


def _shift_box(axis, n, thresh, overlap, V):
    """kt_shift.hpp shift_box: the slab [lo, hi) that leaves the volume when it moves by n voxels along axis"""
    lo, hi = [0, 0, 0], [V, V, V]
    if n >= thresh:
        hi[axis] = n + 1 + overlap
    elif n <= -thresh:
        lo[axis], hi[axis] = (V + (n - overlap), V) if axis < 2 else (V + (n - overlap) - 1, V - 1)
    return lo, hi


def test_meshing_leaves_the_tracker_alone_and_slices_equal_the_operator(built):
    import torch
    import kintinuous_b200 as kb
    from kintinuous_b200 import synth
    rows, cols, V = 240, 320, 256
    frames = [synth.render(k, cols, rows) for k in range(30)]
    runs = {}
    for on in (False, True):
        trk = kb.Tracker(kb.Config.default(rows=rows, cols=cols, vol=V, odometry=0, voxel_shift=2))
        trk.set_slice_processing(True, 8)
        if on:
            trk.set_slice_meshing(True, 8)
        poses, launches, shifted = [], [], []
        for k, (d, c) in enumerate(frames):
            l0 = trk.launch_count()
            p = trk.process_frame(d, c, k)
            launches.append(trk.launch_count() - l0); shifted.append(p.shifted)
            poses.append(bytes(p))
        trk.finalise()
        n = trk.num_slices()
        raw = [_canon(trk.get_slice(i)[0]) for i in range(n)]           # extraction order is unspecified (atomics)
        proc = [trk.get_processed_slice(i).tobytes() for i in range(n)]
        meshes = [trk.get_slice_mesh(i) for i in range(n)] if on else None
        live = trk.live_mesh() if on else None
        if on:
            t, c = trk.export_volume()
            w = list(trk.pose().voxel_wrap)
            final = _mesh(kb, t, c, V, 6.0, w, w, BOXES_FULL(V))
        runs[on] = (poses, launches, shifted, raw, proc, meshes, live, final if on else None)
        if not on:
            with pytest.raises(kb.KtError):
                trk.get_slice_mesh(0)
        trk.close()
    off, on = runs[False], runs[True]
    assert off[0] == on[0]                                                              # poses
    assert len(off[3]) == len(on[3]) and all(np.array_equal(a, b) for a, b in zip(off[3], on[3]))   # raw slices (as sets)
    assert off[4] == on[4]                                                             # processed slices, bit for bit
    quiet = [i for i in range(1, 30) if on[2][i] == 0]
    assert quiet and all(off[1][i] == on[1][i] for i in quiet)                         # launches of a frame without a shift
    meshes, live, final = on[5], on[6], on[7]
    n_shift = len(meshes) - 1
    assert n_shift >= 3
    for got in (meshes[-1], live):
        assert got[0].tobytes() == final[0].tobytes() and np.array_equal(got[1], final[1])
    print(f"tracker: {n_shift} shift slices + FINAL; FINAL mesh {len(final[0])} vertices, {len(final[1])} triangles")
    # every shift slice: replay a lock-step tracker with meshing off, mesh its volume as it was before the frame
    trk = kb.Tracker(kb.Config.default(rows=rows, cols=cols, vol=V, odometry=0, voxel_shift=2))
    si = 0
    for k, (d, c) in enumerate(frames):
        if on[2][k]:
            t, col = trk.export_volume()
            w0 = list(trk.pose().voxel_wrap)
            td, cd = _dev(t, col)
        p = trk.process_frame(d, c, k)
        if not on[2][k]:
            continue
        w1 = list(p.voxel_wrap)
        wrap = list(w0)
        for axis in range(3):
            n = w1[axis] - w0[axis]
            if n == 0:
                continue
            lo, hi = _shift_box(axis, n, 2, 2, V)
            want = kb.ops.mesh_volume(td, cd, V, [6.0] * 3, wrap, wrap, (lo[0], hi[0], lo[1], hi[1], lo[2], hi[2]), 8)
            got = meshes[si]
            assert got[0].tobytes() == want[0].tobytes() and np.array_equal(got[1], want[1]), (k, axis)
            kb.ops.clear_volume(axis, 1 if n < 0 else 0, td, cd, V, wrap[axis], wrap[axis] + n)
            wrap[axis] += n
            si += 1
        torch.cuda.synchronize()
    assert si == n_shift
    trk.close()


def _scene_distance(p):
    """distance (m) to the synthetic scene's surfaces: room walls (seen from inside), sphere, cube"""
    from kintinuous_b200 import synth
    room = np.min(synth.ROOM_HALF - np.abs(p), axis=1)
    sph = np.abs(np.linalg.norm(p - synth.SPHERE_C, axis=1) - synth.SPHERE_R)
    c = (synth.CUBE_LO + synth.CUBE_HI) / 2; h = (synth.CUBE_HI - synth.CUBE_LO) / 2
    q = np.abs(p - c) - h
    cube = np.abs(np.linalg.norm(np.maximum(q, 0), axis=1) + np.minimum(q.max(1), 0))
    return np.minimum(np.abs(room), np.minimum(sph, cube))


def test_real_geometry_and_ply(built, tmp_path):
    import kintinuous_b200 as kb
    from kintinuous_b200 import synth
    trk = kb.Tracker(kb.Config.default(rows=480, cols=640, vol=512, odometry=0))
    trk.set_slice_meshing(True, 8)
    for k in range(72):
        d, c = synth.render(k, 640, 480)
        trk.process_frame(d, c, k)
    trk.finalise()
    meshes = [trk.get_slice_mesh(i) for i in range(trk.num_slices())]
    verts = np.concatenate([m[0] for m in meshes])
    offs = np.cumsum([0] + [len(m[0]) for m in meshes[:-1]])
    tris = np.concatenate([m[1].astype(np.int64) + o for m, o in zip(meshes, offs)])
    assert len(verts) > 50000
    p = np.stack([verts["x"], verts["y"], verts["z"]], -1).astype(np.float64)
    dist = _scene_distance(p) / trk.voxel_size
    q = np.quantile(dist, [0.5, 0.9, 0.99, 0.999])
    print(f"real geometry: {len(meshes)} slices, {len(verts)} vertices, {len(tris)} triangles; distance to the analytic scene in voxels: "
          f"median {q[0]:.3f}, 90 % {q[1]:.3f}, 99 % {q[2]:.3f}, 99.9 % {q[3]:.3f}, max {dist.max():.2f}")
    assert (dist <= 1.5).mean() >= 0.99
    path = str(tmp_path / "mesh.ply")
    trk.save_mesh_ply(path)
    blob = open(path, "rb").read()
    head, body = blob.split(b"end_header\n", 1)
    lines = head.decode().splitlines()
    nv = int([ln for ln in lines if ln.startswith("element vertex")][0].split()[-1])
    nf = int([ln for ln in lines if ln.startswith("element face")][0].split()[-1])
    vdt = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4"), ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    fdt = np.dtype([("n", "u1"), ("i", "<i4", (3,))])
    assert (nv, nf) == (len(verts), len(tris)) and len(body) == nv * vdt.itemsize + nf * fdt.itemsize
    pv = np.frombuffer(body, vdt, nv); pf = np.frombuffer(body, fdt, nf, offset=nv * vdt.itemsize)
    for a, b in (("x", "x"), ("y", "y"), ("z", "z"), ("nx", "nx"), ("ny", "ny"), ("nz", "nz"), ("red", "r"), ("green", "g"), ("blue", "b")):
        assert np.array_equal(pv[a], verts[b]), a
    assert (pf["n"] == 3).all() and np.array_equal(pf["i"], tris)
    trk.close()
