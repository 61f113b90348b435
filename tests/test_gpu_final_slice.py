"""The FINAL slice kt_finalise records (the whole volume, CloudSlice::FINAL) against the whole-volume operators on the tracker's own
volume after a seeded shifting run: its points against kt_op_extract_slice (as sets: the extraction order comes from atomics), its
processed points against kt_op_process_slice of those points, its mesh and mesh keys against kt_op_mesh_volume_keyed, all bit for
bit; and kt_get_live_tsdf, which cuts the same box without recording it."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _canon(p):
    a = np.ascontiguousarray(p).view(np.uint64).reshape(len(p), 4)
    return a[np.lexsort(a.T[::-1])] if len(a) else a


def test_final_slice_equals_the_whole_volume_operators(built):
    import torch
    import kintinuous_b200 as kb
    from kintinuous_b200 import synth
    from kintinuous_b200.binding import POINT_DTYPE
    rows, cols, V, size = 240, 320, 256, 6.0
    trk = kb.Tracker(kb.Config.default(rows=rows, cols=cols, vol=V, odometry=0, voxel_shift=2))
    trk.set_slice_processing(True, 8)
    trk.set_slice_meshing(True, 8)
    for k in range(30):
        d, c = synth.render(k, cols, rows)
        trk.process_frame(d, c, k)
    trk.finalise()
    n = trk.num_slices()
    pts, dim, _ = trk.get_slice(n - 1)
    assert n >= 4 and dim == 7                                                          # shift slices, then FINAL
    proc = trk.get_processed_slice(n - 1)
    verts, tris = trk.get_slice_mesh(n - 1)
    edges, cells = trk.get_slice_mesh_keys(n - 1)
    live = trk.live_tsdf()
    t, col = trk.export_volume()
    w = [int(x) for x in trk.pose().voxel_wrap]
    leaf = trk.voxel_size
    trk.close()
    assert any(w)                                                                       # the volume has moved: wraps are not zero
    td, cd = torch.from_numpy(t).cuda(), torch.from_numpy(col).cuda()
    wrap, box, cap = [x % V for x in w], (0, V, 0, V, 0, V), 3 * rows * cols
    out = torch.zeros(cap * 32, dtype=torch.uint8, device="cuda")
    m = kb.ops.extract_slice(td, [size] * 3, V, out, cap, wrap, cd, box, 1, w)
    want = out[:m * 32].cpu().numpy().view(POINT_DTYPE)
    assert 5000 < m < cap and len(pts) == len(live) == m
    assert np.array_equal(_canon(pts), _canon(want)) and np.array_equal(_canon(live), _canon(want))
    pout = torch.zeros(m * 48, dtype=torch.uint8, device="cuda")
    pn = kb.ops.process_slice(out, m, 8, leaf, pout, m)
    assert len(proc) == pn > 0 and proc.tobytes() == pout[:pn * 48].cpu().numpy().tobytes()
    v, tr, e, k = kb.ops.mesh_volume_keyed(td, cd, V, [size] * 3, wrap, w, box, 8)
    assert len(tr) > 1000
    assert verts.tobytes() == v.tobytes() and np.array_equal(tris, tr)
    assert np.array_equal(edges, e) and np.array_equal(cells, k)
    print(f"FINAL slice: {m} points, {pn} processed, {len(v)} vertices, {len(tr)} triangles; voxel wrap {w}")
