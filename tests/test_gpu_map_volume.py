"""The map volume on the device (kt_mapvol.cu): the store against tests/map_volume_oracle.py rebuilt from the volume exported after every
frame and the planes kt_op_clear_volume zeroes, the map mesh bit for bit, no interference with tracking, determinism, capacity, refusal
and lifecycle, and kt_op_mesh_bricks against kt_op_mesh_volume on a 1024^3 sphere."""
import os
import sys

import numpy as np
import pytest

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tests"))
import map_volume_oracle as mv  # noqa: E402
from test_gpu_mesh import _canon  # noqa: E402

pytestmark = pytest.mark.gpu

ROWS, COLS, V, SIZE = 240, 320, 128, 3.0
# A 3 m volume puts the synthetic scene's sphere, cube and walls near its faces, so that the slabs a shift clears hold surface.  The
# camera goes out and back along x, y and z, then out along x again: that leg re-meshes cells the first one meshed (the R17 case).
LEG, STEP = 20, 0.025          # frames per leg, metres per frame


def _trajectory():
    t, out = np.zeros(3), [np.zeros(3)]
    for axis, sgn in ((0, 1), (0, -1), (1, 1), (1, -1), (2, 1), (2, -1), (0, 1)):
        for _ in range(LEG):
            t = t.copy(); t[axis] += sgn * STEP
            out.append(t)
    return out


def _track(kb, store=None, per_frame=None, act=None, meshing=True):
    """Tracks the out-and-back stream; store = max_bricks (None: off).  per_frame(trk, k, wrap_before, pose) after every frame."""
    from kintinuous_b200 import synth
    trk = kb.Tracker(kb.Config.default(rows=ROWS, cols=COLS, vol=V, volume_size=SIZE, odometry=0, voxel_shift=2))
    if meshing:
        trk.set_slice_meshing(True, 8)
    if store is not None:
        trk.set_map_volume(True, store)
    poses, launches, shifted = [], [], []
    traj = _trajectory()
    for k, t in enumerate(traj):
        if act is not None and k == len(traj) // 2:
            act(trk)
        d, c = synth.render_at(np.eye(3), t, COLS, ROWS)
        before = tuple(trk.pose().voxel_wrap)
        if per_frame is not None:
            per_frame(trk, k, before, None)
        l0 = trk.launch_count()
        p = trk.process_frame(d, c, k)
        launches.append(trk.launch_count() - l0)
        shifted.append(sum(a != b for a, b in zip(p.voxel_wrap, before)))
        poses.append(bytes(p) + trk.trace().tobytes())        # the pose and the odometry trace of the frame
    return trk, poses, launches, shifted


def _cleared_planes(kb, torch, axis, back, cur, delta):
    x = torch.full((V ** 3,), 7, dtype=torch.int16, device="cuda"); y = torch.full((V ** 3 * 4,), 9, dtype=torch.uint8, device="cuda")
    kb.ops.clear_volume(axis, back, x, y, V, cur, delta)
    zt = (x.view(V, V, V) == 0)
    dims = {0: (0, 1), 1: (0, 2), 2: (1, 2)}[axis]
    return torch.nonzero(zt.all(dim=dims[1]).all(dim=dims[0])).flatten().cpu().numpy()


class _Oracle:
    """Rebuilds the store from the volume as it was before every frame and the wrap that frame moved to."""

    def __init__(self, kb, torch, capacity=None):
        self.kb, self.torch = kb, torch
        self.store = mv.Store(capacity)
        self.vol = None
        self.clears = 0

    def before(self, trk, k, wrap, _):
        self.vol = trk.export_volume(); self.wrap = wrap

    def after(self, trk):
        new = tuple(trk.pose().voxel_wrap)
        t, c = self.vol[0].copy(), self.vol[1].copy()
        w = list(self.wrap)
        for axis in range(3):
            if new[axis] == w[axis]:
                continue
            planes = _cleared_planes(self.kb, self.torch, axis, int(new[axis] < w[axis]), w[axis], new[axis])
            g, tt, cc, idx = mv.cleared_voxels(t, c, V, axis, planes, w)
            self.store.clear(g, tt, cc)
            t[idx] = 0; c[idx] = 0
            self.clears += 1
            w[axis] = new[axis]


def _run_with_oracle(kb, torch, store, act=None):
    orc = _Oracle(kb, torch, None if store is None else store)
    state = {"trk": None}

    def per_frame(trk, k, wrap, _):
        if state["trk"] is not None:
            orc.after(trk)
        state["trk"] = trk
        orc.before(trk, k, wrap, None)
    trk, poses, launches, shifted = _track(kb, store=store, per_frame=per_frame, act=act)
    orc.after(trk)
    return trk, orc, poses, launches, shifted


def _stores_equal(trk, store):
    k, t, c = trk.map_volume_bricks()
    wk, wt, wc = store.sorted()
    assert np.array_equal(k, wk)
    assert np.array_equal(t, wt) and np.array_equal(c, wc)
    return len(k)


def test_no_shift_map_mesh_is_the_live_mesh(built):
    import kintinuous_b200 as kb
    from kintinuous_b200 import synth
    trk = kb.Tracker(kb.Config.default(rows=ROWS, cols=COLS, vol=V, odometry=0))
    trk.set_map_volume(True, 4096)
    for k in range(12):                                     # weights reach 8: the cull-8 mesh is not empty
        d, c = synth.render(k, COLS, ROWS)
        p = trk.process_frame(d, c, k)
        assert tuple(p.voxel_wrap) == (0, 0, 0)
    for cull in (1, 8):
        trk.set_slice_meshing(False, cull)
        lv, lt = trk.live_mesh()
        gv, gt, rep = trk.global_mesh(cull)
        assert len(lt) > 100 and rep["store_bricks"] == 0 and rep["bricks"] == rep["live_bricks"] > 0
        assert gv.tobytes() == lv.tobytes() and np.array_equal(gt, lt), cull
    trk.close()


def test_shifting_run_store_and_map_mesh_against_the_oracle(built, tmp_path):
    import torch
    import kintinuous_b200 as kb
    trk, orc, poses, launches, shifted = _run_with_oracle(kb, torch, 1 << 16)
    wraps = [tuple(trk.pose().voxel_wrap)]
    assert orc.clears >= 6 and sum(shifted) == orc.clears
    n = _stores_equal(trk, orc.store)
    assert n > 0 and trk.map_volume_info() == (n, 1 << 16, False)
    # the map mesh: the oracle's field S meshed by kt_op_mesh_bricks, and by the numpy restatement
    gv, gt, rep = trk.global_mesh(8)
    t, c = trk.export_volume()
    T, C, o = mv.merged(orc.store, t, c, V, wraps[0])
    keys, bt, bc = mv.box_bricks(T, C, o)
    size = SIZE
    ov, ot = kb.ops.mesh_bricks(keys, bt, bc, [size] * 3, V, 8)
    assert gv.tobytes() == ov.tobytes() and np.array_equal(gt, ot)
    nv, nt, own = mv.mesh_global(T, C, o, np.float32(size) / np.float32(V), V, 8)
    assert np.array_equal(gt, nt)
    for f in ("nx", "ny", "nz"):
        np.testing.assert_allclose(gv[f], nv[f], atol=2e-5)
    for f in ("r", "g", "b", "a"):
        assert np.array_equal(gv[f], nv[f])
    for f in ("x", "y", "z"):
        np.testing.assert_allclose(gv[f], nv[f], atol=1e-5)
    # the R17 case is exercised: slices re-meshed cells; the map mesh has no open edge the oracle's has not
    _, _, wrep = trk.map_mesh(0, True)
    print("weld:", wrep, "map volume:", rep)
    assert wrep["repeated_cells"] > 0
    assert len(mv.open_edges(gt)) == len(mv.open_edges(nt))
    assert rep["output_verts"] == len(gv) and rep["output_tris"] == len(gt) and rep["store_bricks"] == n
    trk.save_global_mesh_ply(str(tmp_path / "g.ply"), 8)
    blob = (tmp_path / "g.ply").read_bytes()
    assert f"element vertex {len(gv)}\n".encode() in blob and f"element face {len(gt)}\n".encode() in blob
    # lifecycle: the whole map survives kt_finalise, reset empties the store, disabling frees it
    trk.finalise()
    fv, ft, _ = trk.global_mesh(8)
    assert fv.tobytes() == gv.tobytes() and np.array_equal(ft, gt)
    trk.reset()
    assert trk.map_volume_info()[0] == 0
    trk.set_map_volume(False)
    with pytest.raises(kb.KtError, match="error -3"):
        trk.map_volume_info()
    trk.close()


def test_no_interference_determinism_and_launches(built):
    import kintinuous_b200 as kb
    off, off_poses, off_launches, shifted = _track(kb)
    mid = {}

    def act(trk):
        mid["mesh"] = trk.global_mesh(8)
    on, on_poses, on_launches, _ = _track(kb, store=1 << 16, act=act)
    again, again_poses, _, _ = _track(kb, store=1 << 16)
    assert on_poses == off_poses == again_poses and any(shifted)
    for k in range(len(on_launches)):                         # three launches per cleared slab, nothing on other frames
        assert on_launches[k] == off_launches[k] + 3 * shifted[k], k
    assert on.num_slices() == off.num_slices() > 0
    for i in range(on.num_slices()):
        assert np.array_equal(_canon(on.get_slice(i)[0]), _canon(off.get_slice(i)[0]))      # extraction order is unspecified
        a, b = on.get_slice_mesh(i), off.get_slice_mesh(i)
        assert a[0].tobytes() == b[0].tobytes() and np.array_equal(a[1], b[1])
    ka, kb_ = on.map_volume_bricks(), again.map_volume_bricks()
    assert all(np.array_equal(x, y) for x, y in zip(ka, kb_))
    ma, mb = on.global_mesh(8), again.global_mesh(8)
    assert ma[0].tobytes() == mb[0].tobytes() and np.array_equal(ma[1], mb[1]) and len(mid["mesh"][1]) > 0
    off.close(); on.close(); again.close()


def test_small_capacity_and_oversized_store(built):
    import torch
    import kintinuous_b200 as kb
    ref, ref_poses, _, _ = _track(kb, meshing=False)
    cap = 24
    trk, orc, poses, _, _ = _run_with_oracle(kb, torch, cap)
    assert poses == ref_poses
    n = _stores_equal(trk, orc.store)
    assert orc.store.full and trk.map_volume_info() == (n, cap, True) and n <= cap
    assert trk.global_mesh(8)[2]["store_full"] == 1
    trk.close()

    def huge(t):
        with pytest.raises(kb.KtError, match="error -2"):
            t.set_map_volume(True, 1 << 30)                 # 3 TB of bricks: refused, and nothing changes
        with pytest.raises(kb.KtError, match="error -3"):
            t.map_volume_info()
    big, big_poses, _, _ = _track(kb, meshing=False, act=huge)
    assert big_poses == ref_poses
    ref.close(); big.close()


def test_mesh_bricks_equals_the_volume_mesh_at_1024(built):
    import torch
    import kintinuous_b200 as kb
    N, size = 1024, 6.0
    ar = torch.arange(N, device="cuda", dtype=torch.float32)
    z, y, x = ar.view(N, 1, 1), ar.view(1, N, 1), ar.view(1, 1, N)
    d = torch.sqrt((x - 0.45 * N) ** 2 + (y - 0.52 * N) ** 2 + (z - 0.5 * N) ** 2) - 0.3 * N
    tsdf = torch.trunc(torch.clamp(d / 4.0, -1, 1) * 32767).to(torch.int16)
    del d
    g = torch.Generator(device="cuda"); g.manual_seed(5)
    col = torch.randint(0, 256, (N, N, N, 4), dtype=torch.uint8, device="cuda", generator=g)
    col[..., 3] = 20
    vv, vt = kb.ops.mesh_volume(tsdf, col, N, [size] * 3, (0, 0, 0), (0, 0, 0), (0, N, 0, N, 0, N), 8)
    nb = N // 8
    bt = tsdf.view(nb, 8, nb, 8, nb, 8).permute(0, 2, 4, 1, 3, 5).contiguous()
    bc = col.view(nb, 8, nb, 8, nb, 8, 4).permute(0, 2, 4, 1, 3, 5, 6).contiguous()
    del tsdf, col
    # only the bricks with a surface voxel: the others cannot change the mesh
    keep = ((bt != 32767).flatten(3).any(-1)).flatten()
    bz, by, bx = torch.meshgrid(*[torch.arange(nb, device="cuda", dtype=torch.int64)] * 3, indexing="ij")
    bias = 1 << 20
    keys = (((bz + bias) << 42) | ((by + bias) << 21) | (bx + bias)).flatten()[keep].contiguous()
    bt = bt.view(-1, 8, 8, 8)[keep].contiguous(); bc = bc.view(-1, 8, 8, 8, 4)[keep].contiguous()
    bv, btri = kb.ops.mesh_bricks(keys, bt, bc, [size] * 3, N, 8)
    print(f"1024^3 sphere: {len(keys)} bricks, {len(bv)} vertices, {len(btri)} triangles")
    assert len(vt) > 1000000
    assert bv.tobytes() == vv.tobytes() and np.array_equal(btri, vt)
    # unsorted keys are refused
    with pytest.raises(kb.KtError, match="error -1"):
        kb.ops.mesh_bricks(keys.flip(0).contiguous(), bt, bc, [size] * 3, N, 8)
