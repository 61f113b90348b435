"""The map volume's restore on the device (kt_set_map_volume_restore, mapvol_restore_kernel): every voxel of every frame against a lock-step
replay (tests/map_volume_restore_oracle.py's store -> clear -> restore per shifted axis, then kt_op_integrate at the tracker's own
integration pose), the store and the map mesh at the end, the property the feature exists for (a revisit never lowers a stored weight), launches,
determinism and the setting's lifecycle."""
import os
import sys

import numpy as np
import pytest

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tests"))
import map_volume_oracle as mv  # noqa: E402
import map_volume_restore_oracle as mr  # noqa: E402
from test_gpu_map_volume import COLS, LEG, ROWS, SIZE, STEP, V, _cleared_planes, _stores_equal, _trajectory  # noqa: E402

pytestmark = pytest.mark.gpu


def _stream():
    """test_gpu_map_volume's out-and-back trajectory, then a diagonal leg on which x and y shift in the same frames."""
    traj = _trajectory()
    t = traj[-1]
    for _ in range(LEG):
        t = t + np.array([STEP, STEP, 0.0])
        traj.append(t)
    return traj


_FRAMES = {}


def _frame(t):
    from kintinuous_b200 import synth
    key = tuple(np.round(t, 9))
    if key not in _FRAMES:
        _FRAMES[key] = synth.render_at(np.eye(3), t, COLS, ROWS)
    return _FRAMES[key]


def _track(kb, store=1 << 16, restore=True, before=None, after=None, act=None):
    """Tracks the stream with the map volume on (store = max_bricks) and restore set; before(trk, k) / after(trk, k, d, c) around each
    frame, act(trk, k) before frame k.  Returns (tracker, poses + traces, launches, shifted axes) per frame."""
    trk = kb.Tracker(kb.Config.default(rows=ROWS, cols=COLS, vol=V, volume_size=SIZE, odometry=0, voxel_shift=2))
    if store is not None:
        trk.set_map_volume(True, store)
        if restore:
            trk.set_map_volume_restore(True)
    poses, launches, shifted = [], [], []
    for k, t in enumerate(_stream()):
        if act is not None:
            act(trk, k)
        d, c = _frame(t)
        w0 = tuple(trk.pose().voxel_wrap)
        if before is not None:
            before(trk, k)
        l0 = trk.launch_count()
        p = trk.process_frame(d, c, k)
        launches.append(trk.launch_count() - l0)
        shifted.append(sum(a != b for a, b in zip(p.voxel_wrap, w0)))
        poses.append(bytes(p) + trk.trace().tobytes())
        if after is not None:
            after(trk, k, d, c)
    return trk, poses, launches, shifted


class _Replay:
    """Before each frame the volume and wrap are exported; after it, the oracle shifts that volume axis by axis (store -> clear ->
    restore) and integrates the frame with kt_op_integrate at the tracker's integration pose.  The result must be the tracker's volume."""

    def __init__(self, kb, torch, restore, capacity=None):
        self.kb, self.torch, self.restore = kb, torch, restore
        self.store = mv.Store(capacity)
        self.shifts = self.restored = 0

    def before(self, trk, k):
        self.vol = trk.export_volume(); self.wrap = list(trk.pose().voxel_wrap)

    def after(self, trk, k, d, c):
        torch, kb = self.torch, self.kb
        from kintinuous_b200 import synth
        new = tuple(trk.pose().voxel_wrap)
        t, col = self.vol[0].copy(), self.vol[1].copy()
        w = self.wrap
        for axis in range(3):
            if new[axis] == w[axis]:
                continue
            planes = _cleared_planes(kb, torch, axis, int(new[axis] < w[axis]), w[axis], new[axis])
            w = mr.shift_axis(self.store, t, col, V, axis, planes, w, new[axis] - w[axis], self.restore)
            if self.restore:
                self.restored += int(mr.restore(self.store, mv.cleared_voxels(t, col, V, axis, planes, w)[0])[2].sum())
            self.shifts += 1
        Rinv, tint, wint = trk.last_integrate()
        intr = np.array(synth.intrinsics(COLS, ROWS), np.float32)
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()        # noqa: E731
        ts, cs = dev(t.reshape(-1)), dev(col.reshape(-1))
        nm = dev(trk.download_map(1, 0).reshape(3 * ROWS, COLS))
        ds = torch.zeros((ROWS, COLS), dtype=torch.float32, device="cuda")
        kb.ops.integrate(dev(d.view(np.int16)), ROWS, COLS, intr, [SIZE] * 3, Rinv, tint, trk.trunc_dist, ts, cs, V, wint, dev(c), nm,
                         trk.cfg.angle_color, ds)
        torch.cuda.synchronize()
        gt, gc = trk.export_volume()
        rt, rc = ts.cpu().numpy().reshape(V, V, V), cs.cpu().numpy().reshape(V, V, V, 4)
        assert np.array_equal(gt, rt), (k, "tsdf", int((gt != rt).sum()))
        assert np.array_equal(gc, rc), (k, "colour / weight", int((gc != rc).any(-1).sum()))


def _exact_run(kb, torch, restore, capacity=1 << 16):
    rp = _Replay(kb, torch, restore, None if capacity == 1 << 16 else capacity)
    trk, poses, _, shifted = _track(kb, store=capacity, restore=restore, before=rp.before, after=rp.after)
    assert rp.shifts == sum(shifted) >= 6
    return trk, rp


def test_every_voxel_of_every_frame_equals_the_replay(built):
    import torch
    import kintinuous_b200 as kb
    # the replay itself first, on the store-only path: a failure below then points at the restore
    off, rp_off = _exact_run(kb, torch, False)
    _stores_equal(off, rp_off.store)
    off.close()
    trk, rp = _exact_run(kb, torch, True)
    print(f"restore: {rp.shifts} cleared slabs, {rp.restored} voxels restored, {len(rp.store.bricks)} bricks stored")
    assert rp.restored > 1000
    n = _stores_equal(trk, rp.store)
    assert n > 0 and trk.map_volume_info() == (n, 1 << 16, False)
    # the map mesh: kt_op_mesh_bricks over the oracle's field S (the store merged with the live volume)
    gv, gt, rep = trk.global_mesh(8)
    t, c = trk.export_volume()
    T, C, o = mv.merged(rp.store, t, c, V, tuple(trk.pose().voxel_wrap))
    keys, bt, bc = mv.box_bricks(T, C, o)
    ov, ot = kb.ops.mesh_bricks(keys, bt, bc, [SIZE] * 3, V, 8)
    assert len(gt) > 0 and gv.tobytes() == ov.tobytes() and np.array_equal(gt, ot)
    trk.close()


def test_a_small_store_stays_exact(built):
    import torch
    import kintinuous_b200 as kb
    cap = 24
    trk, rp = _exact_run(kb, torch, True, capacity=cap)
    n = _stores_equal(trk, rp.store)
    assert rp.store.full and trk.map_volume_info() == (n, cap, True)
    trk.close()


def _weight_falls(kb, restore):
    """Stored voxels whose weight is lower than in the previous frame's store, summed over the stream."""
    prev = {}
    falls = [0]

    def after(trk, k, d, c):
        keys, _, col = trk.map_volume_bricks()
        w = col[..., 3]
        for i, key in enumerate(keys.tolist()):
            if key in prev:
                falls[0] += int((w[i] < prev[key]).sum())
            prev[key] = w[i].copy()
    trk, _, _, _ = _track(kb, restore=restore, after=after)
    trk.close()
    return falls[0], len(prev)


def test_a_revisit_never_lowers_a_stored_weight(built):
    import kintinuous_b200 as kb
    off, n_off = _weight_falls(kb, False)
    on, n_on = _weight_falls(kb, True)
    print(f"stored voxels whose weight fell: {off} with restore off ({n_off} bricks), {on} with it on ({n_on} bricks)")
    assert off > 0 and on == 0


def test_launches_determinism_and_lifecycle(built):
    import kintinuous_b200 as kb
    ref, ref_poses, ref_launches, ref_shifted = _track(kb, restore=False)
    on, on_poses, on_launches, on_shifted = _track(kb)
    again, again_poses, _, _ = _track(kb)
    # launches: store-only frames are base + per_slab * slabs; with restore exactly one more per slab, nothing more elsewhere
    assert sum(ref_shifted) > 0 and sum(on_shifted) > 0 and on_launches[0] == ref_launches[0]
    base = {ref_launches[k] for k in range(1, len(ref_launches)) if ref_shifted[k] == 0}
    assert len(base) == 1, base
    b = base.pop()
    per = {(ref_launches[k] - b) / ref_shifted[k] for k in range(1, len(ref_launches)) if ref_shifted[k]}
    assert len(per) == 1, per
    s = per.pop()
    for k in range(1, len(on_launches)):
        assert on_launches[k] == b + (s + 1) * on_shifted[k], (k, on_launches[k], on_shifted[k])
    # two restore-on runs: poses, traces, volume, store and map mesh bit for bit
    assert on_poses == again_poses
    for x, y in zip(on.export_volume(), again.export_volume()):
        assert np.array_equal(x, y)
    assert all(np.array_equal(x, y) for x, y in zip(on.map_volume_bricks(), again.map_volume_bricks()))
    ma, mb = on.global_mesh(8), again.global_mesh(8)
    assert len(ma[1]) > 0 and ma[0].tobytes() == mb[0].tobytes() and np.array_equal(ma[1], mb[1])
    # the setting survives kt_reset: the whole stream again after a reset is the restore-on run
    on.reset()
    for k, t in enumerate(_stream()):
        d, c = _frame(t)
        p = on.process_frame(d, c, k)
        assert bytes(p) + on.trace().tobytes() == on_poses[k], k
    again.close(); on.close()

    def toggle(trk, k):
        if k == 1:                                              # before the first shift: on, then off again
            trk.set_map_volume_restore(True); trk.set_map_volume_restore(False)
    tog, tog_poses, _, _ = _track(kb, restore=False, act=toggle)
    assert tog_poses == ref_poses
    tog.close()

    def replace(trk, k):
        if k == 0:                                              # a replacing store keeps the setting; disabling the store clears it
            trk.set_map_volume(True, 1 << 16)
    rep, rep_poses, _, _ = _track(kb, act=replace)
    assert rep_poses == on_poses
    rep.set_map_volume(False)
    with pytest.raises(kb.KtError, match="error -3"):
        rep.set_map_volume_restore(True)
    rep.close()

    def cleared(trk, k):
        if k == 0:
            trk.set_map_volume(False); trk.set_map_volume(True, 1 << 16)
    clr, clr_poses, _, _ = _track(kb, act=cleared)
    assert clr_poses == ref_poses and ref_poses != on_poses
    clr.close(); ref.close()
    # off by default, and refused while the map volume is off
    bare = kb.Tracker(kb.Config.default(rows=ROWS, cols=COLS, vol=V, volume_size=SIZE, odometry=0, voxel_shift=2))
    with pytest.raises(kb.KtError, match="error -3"):
        bare.set_map_volume_restore(True)
    bare.close()
