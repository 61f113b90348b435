"""The map volume's restore restated in numpy (tests/map_volume_restore_oracle.py): once a shift has cleared its planes, every voxel of
them whose global voxel lies in a stored brick with W != 0 takes the stored value, under the wrap after the shift.  A surface that leaves and comes
back resumes with its bits and weights, the plane a clear reaches beyond those that leave comes back in the same step, free space
outside stored bricks stays cleared, a clear refused for capacity restores nothing, and the next axis's store of restored voxels changes
nothing."""
import copy
import os
import sys

import numpy as np

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tests"))
import map_volume_oracle as mv  # noqa: E402
import map_volume_restore_oracle as mr  # noqa: E402
from oracle import mesh_oracle as mo  # noqa: E402
from test_map_volume_oracle import _sphere  # noqa: E402

V = 32


def _global_planes(axis, planes, wrap):
    """Global coordinate along axis of storage planes at a signed wrap."""
    w = int(wrap[axis])
    return (np.asarray(planes, np.int64) - w % V) % V + w


def _stored_mask(store, axis, planes, wrap):
    """[z, y, x] mask over the whole volume: storage voxels of `planes` whose global voxel at `wrap` lies in a stored brick."""
    m = np.zeros((V, V, V), bool)
    g, _, _, idx = mv.cleared_voxels(np.zeros((V, V, V), np.int16), np.zeros((V, V, V, 4), np.uint8), V, axis, planes, wrap)
    b = g >> 3
    keys = mv.brick_key(b[:, 0], b[:, 1], b[:, 2])
    m[idx] = np.isin(keys, np.array(list(store.bricks), np.int64))
    return m


def _plane_sel(axis, planes):
    sel = [slice(None)] * 3
    sel[2 - axis] = np.asarray(planes)
    return tuple(sel)


def _out_and_back(axis, n, centre, capacity=None):
    """A sphere near the face the first shift (n along axis, either sign) clears; out by n and back by -n with restore.  Returns the
    original volume, the volume after, the store, the planes of both clears and the plane set after the first step."""
    t, c = _sphere(V, centre, 5.2, seed=axis + (n > 0))
    orig = (t.copy(), c.copy())
    st = mv.Store(capacity)
    wrap = [0, 0, 0]
    p1 = mr.clear_planes(axis, int(n < 0), V, 0, n)
    wrap = mr.shift_axis(st, t, c, V, axis, p1, wrap, n, True)
    mid = (t.copy(), c.copy())
    p2 = mr.clear_planes(axis, int(n > 0), V, wrap[axis], 0)
    wrap = mr.shift_axis(st, t, c, V, axis, p2, wrap, -n, True)
    assert wrap == [0, 0, 0]
    return orig, (t, c), st, p1, p2, mid


def _check_returned(orig, now, st, axis, planes):
    """The planes are back: stored bricks' voxels equal the original, every other voxel of the planes is zero, the rest is untouched."""
    (t0, c0), (t, c) = orig, now
    m = _stored_mask(st, axis, planes, (0, 0, 0))
    sel = np.zeros((V, V, V), bool); sel[_plane_sel(axis, planes)] = True
    assert np.array_equal(t[m], t0[m]) and np.array_equal(c[m], c0[m])
    assert not t[sel & ~m].any() and not c[sel & ~m].any()
    assert np.array_equal(t[~sel], t0[~sel]) and np.array_equal(c[~sel], c0[~sel])
    # the planes held both: surface bricks that came back, and observed free space of bricks without a surface that did not
    assert (m & (c0[..., 3] != 0)).sum() > 100 and (sel & ~m & (c0[..., 3] != 0)).sum() > 100
    return m


def test_out_along_x_and_back_restores_the_stored_surface_bricks():
    n = 6
    orig, now, st, p1, p2, _ = _out_and_back(0, n, (6.3, 16.1, 15.7))
    assert np.array_equal(p1, np.arange(n + 1)) and np.array_equal(p2, np.arange(n + 1))
    _check_returned(orig, now, st, 0, np.arange(n + 1))
    # the stored bricks are exactly those with a surface voxel in the planes the first clear reached
    t0, c0 = orig
    g, tt, cc, _ = mv.cleared_voxels(t0, c0, V, 0, p1, (0, 0, 0))
    surf = (cc[:, 3] != 0) & (tt != mo.DIVISOR)
    b = g[surf] >> 3
    assert set(st.bricks) == {int(k) for k in np.unique(mv.brick_key(b[:, 0], b[:, 1], b[:, 2]))}


def test_x_over_clear_comes_back_in_the_same_step():
    """n = 2 clears 3 planes (|n| + 1 <= round_up16(|n|)): storage plane 2 is global x = 2 before and after the shift, so the restore puts
    its surface back at once and only planes 0, 1 (global 32, 33, never stored) stay cleared.  At n = 16, Q13 clears exactly the 16
    planes that leave, and nothing comes back."""
    t0, c0 = _sphere(V, (5.3, 16.1, 15.7), 5.2)
    for restore in (False, True):
        t, c = t0.copy(), c0.copy()
        st = mv.Store()
        planes = mr.clear_planes(0, 0, V, 0, 2)
        assert np.array_equal(planes, [0, 1, 2])
        assert np.array_equal(_global_planes(0, planes, (2, 0, 0)), [32, 33, 2])
        mr.shift_axis(st, t, c, V, 0, planes, [0, 0, 0], 2, restore)
        assert not t[:, :, :2].any() and not c[:, :, :2].any()
        m = _stored_mask(st, 0, [2], (2, 0, 0))
        assert m.sum() > 100
        if restore:
            assert np.array_equal(t[m], t0[m]) and np.array_equal(c[m], c0[m]) and not t[:, :, 2][~m[:, :, 2]].any()
        else:
            assert not t[:, :, 2].any() and not c[:, :, 2].any()
    t, c = t0.copy(), c0.copy()
    st = mv.Store()
    planes = mr.clear_planes(0, 0, V, 0, 16)
    assert np.array_equal(planes, np.arange(16))
    mr.shift_axis(st, t, c, V, 0, planes, [0, 0, 0], 16, True)
    assert len(st.bricks) > 0 and not t[:, :, :16].any() and not c[:, :, :16].any()


def test_y_and_z_both_directions():
    """Forward (n > 0) clears base .. base + n, back (n < 0) base - |n| .. base: the plane below the leaving slab, like the ZMinus slab
    of Q12.  Out and back, each direction and axis, the planes are the stored surface again."""
    for axis in (1, 2):
        for n in (3, -3):
            centre = [16.1, 15.7, 16.3]
            centre[axis] = 5.3 if n > 0 else V - 6.3
            orig, now, st, p1, p2, mid = _out_and_back(axis, n, tuple(centre))
            want = np.arange(4) if n > 0 else np.array([V - 3, V - 2, V - 1, 0])
            assert np.array_equal(np.sort(p1), np.sort(want)) and np.array_equal(np.sort(p2), np.sort(want)), (axis, n, p1, p2)
            # after the first step the planes that left are empty; the plane that stays (global 3 forward, beside the sphere; global 0
            # back, on the far face) holds its stored bricks
            keep = p1[-1] if n > 0 else 0
            w1 = [n if a == axis else 0 for a in range(3)]
            assert _global_planes(axis, [keep], w1)[0] == max(n, 0)
            leaving = [p for p in p1 if p != keep]
            assert not mid[0][_plane_sel(axis, leaving)].any() and not mid[1][_plane_sel(axis, leaving)].any()
            m = _stored_mask(st, axis, [keep], w1)
            assert np.array_equal(mid[0][m], orig[0][m]) and not mid[1][_plane_sel(axis, [keep])][~m[_plane_sel(axis, [keep])]].any()
            assert m.any() == (n > 0)
            _check_returned(orig, now, st, axis, want)


def test_a_clear_refused_for_capacity_restores_nothing():
    t0, c0 = _sphere(V, (6.3, 16.1, 15.7), 5.2)
    full = _out_and_back(0, 6, (6.3, 16.1, 15.7))[2]
    k = len(full.bricks)
    assert k > 2
    orig, (t, c), st, p1, _, _ = _out_and_back(0, 6, (6.3, 16.1, 15.7), capacity=k - 1)
    assert st.full and not st.bricks
    sel = _plane_sel(0, p1)
    assert not t[sel].any() and not c[sel].any()
    assert np.array_equal(orig[0], t0) and orig[0][sel].any()


def test_the_next_axis_stores_restored_voxels_unchanged():
    """x and y shift in one step: the y store reads voxels the x restore has just written (the x over-clear plane meets the y slab), and
    every restored voxel's stored value is what it was."""
    t, c = _sphere(V, (6.1, 6.3, 15.7), 5.5)
    st = mv.Store()
    wrap = [0, 0, 0]
    px = mr.clear_planes(0, 0, V, 0, 2)
    wrap = mr.shift_axis(st, t, c, V, 0, px, wrap, 2, True)
    g, _, _, _ = mv.cleared_voxels(t, c, V, 0, px, wrap)
    rt, rc, m = mr.restore(st, g)
    R = g[m]
    before = copy.deepcopy(st.bricks)
    py = mr.clear_planes(1, 0, V, 0, 2)
    both = np.isin(R[:, 1], _global_planes(1, py, wrap)).sum()        # restored voxels in the planes the y clear reaches
    assert m.sum() > 100 and both > 10
    mr.shift_axis(st, t, c, V, 1, py, wrap, 2, True)
    t2, c2, m2 = mr.restore(st, R)
    assert m2.all() and np.array_equal(t2, rt[m]) and np.array_equal(c2, rc[m])
    assert set(before) <= set(st.bricks)
