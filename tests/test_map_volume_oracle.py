"""The map volume's contract restated in numpy (tests/map_volume_oracle.py): the store keeps each global voxel's latest observation, the
map mesh of a volume that never shifted is the volume's mesh, and where two slices disagree at their shared plane the slice meshes
leave a seam open (DESIGN.md R17) while the map mesh over the one field does not."""
import os
import sys

import numpy as np

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tests"))
import map_volume_oracle as mv  # noqa: E402
from oracle import mesh_oracle as mo  # noqa: E402
from weld_oracle import keyed, weld  # noqa: E402

V, SIZE = 32, 1.5


def _sphere(V, c, r, seed=0):
    z, y, x = np.meshgrid(*[np.arange(V)] * 3, indexing="ij")
    d = np.sqrt((x - c[0]) ** 2 + (y - c[1]) ** 2 + (z - c[2]) ** 2) - r
    col = np.random.default_rng(seed).integers(0, 256, (V, V, V, 4), dtype=np.uint8)
    return mo.sdf_volume(d.astype(np.float32), color=col)


def test_latest_observation_wins():
    st = mv.Store()
    g = np.array([[0, 0, 0], [1, 0, 0], [9, 0, 0], [-1, 0, 0]])
    st.clear(g, np.array([-5, 7, 32767, 3], np.int16), np.array([[1, 2, 3, 4], [5, 6, 7, 8], [1, 1, 1, 9], [0, 0, 0, 0]], np.uint8))
    k0 = int(mv.brick_key(0, 0, 0))
    assert set(st.bricks) == {k0}                         # (9, 0, 0) is free space only, (-1, 0, 0) unobserved: no brick
    t, c = st.bricks[k0]
    assert t[0, 0, 0] == -5 and t[0, 0, 1] == 7 and tuple(c[0, 0, 1]) == (5, 6, 7, 8)
    # a later clear: free space observed at (0, 0, 0) overwrites the surface; an unobserved voxel changes nothing
    st.clear(np.array([[0, 0, 0], [1, 0, 0]]), np.array([32767, 0], np.int16), np.array([[9, 9, 9, 2], [0, 0, 0, 0]], np.uint8))
    t, c = st.bricks[k0]
    assert t[0, 0, 0] == 32767 and tuple(c[0, 0, 0]) == (9, 9, 9, 2) and t[0, 0, 1] == 7
    # capacity: a clear whose new bricks do not all fit creates none, existing bricks are still updated
    st = mv.Store(capacity=2)
    st.clear(np.array([[0, 0, 0], [8, 0, 0], [16, 0, 0]]), np.zeros(3, np.int16), np.full((3, 4), 5, np.uint8))
    assert st.full and not st.bricks
    st.clear(np.array([[0, 0, 0], [8, 0, 0]]), np.zeros(2, np.int16), np.full((2, 4), 5, np.uint8))
    assert len(st.bricks) == 2


def test_no_shift_map_mesh_is_the_volume_mesh():
    t, c = _sphere(V, (15.3, 16.1, 14.7), 9.2)
    for cull in (1, 8):
        want_v, want_t, want_o = mo.mesh(t, c, V, SIZE, (0, 0, 0), (0, 0, 0), (0, V, 0, V, 0, V), cull, return_owners=True)
        T, C, o = mv.merged(mv.Store(), t, c, V, (0, 0, 0))
        v, tt, own = mv.mesh_global(T, C, o, np.float32(SIZE) / np.float32(V), V, cull)
        assert np.array_equal(tt, want_t) and np.array_equal(own, want_o)
        for f in ("nx", "ny", "nz", "r", "g", "b", "a"):
            assert np.array_equal(v[f], want_v[f]), f
        for f in ("x", "y", "z"):
            np.testing.assert_allclose(v[f], want_v[f], atol=2e-6)


def test_the_map_mesh_closes_the_seam_the_slice_meshes_leave():
    """Slice 1 is meshed from field A and cleared (x < CUT), the surface then moves and slice 2 is field B (x >= CUT - 1): per-box meshes
    disagree at the shared plane; S holds A's cleared planes and B where it is observed, one field, and its mesh is closed."""
    CUT = 16
    ta, ca = _sphere(V, (15.3, 16.1, 14.7), 9.2, seed=1)
    tb, cb = _sphere(V, (15.8, 16.1, 14.7), 9.7, seed=2)
    cell = np.float32(SIZE) / np.float32(V)
    m1 = keyed(ta, ca, V, SIZE, (0, 0, 0), (0, 0, 0), (0, CUT, 0, V, 0, V))
    m2 = keyed(tb, cb, V, SIZE, (0, 0, 0), (0, 0, 0), (CUT - 1, V, 0, V, 0, V))
    wv, wt, we, wc, stats = weld([m1, m2])
    ekey = lambda e: ((e[:, 2] * 1000 + e[:, 1]) * 1000 + e[:, 0]) * 3 + e[:, 3]  # noqa: E731
    seam = mv.open_edges(wt, ekey(we))
    assert len(seam) > 0                                   # R17: the welded slice meshes are open at the cut
    # the map field: A's planes x < CUT kept at the clear, then B observed only from CUT on (the cleared planes have W = 0 in the volume)
    st = mv.Store()
    g, t0, c0, _ = mv.cleared_voxels(ta, ca, V, 0, np.arange(CUT), (0, 0, 0))
    st.clear(g, t0, c0)
    tb2, cb2 = tb.copy(), cb.copy()
    tb2[:, :, :CUT] = 0; cb2[:, :, :CUT] = 0
    T, C, o = mv.merged(st, tb2, cb2, V, (0, 0, 0))
    v, t, own = mv.mesh_global(T, C, o, cell, V)
    assert len(t) > 0 and len(mv.open_edges(t)) == 0       # one field: a closed surface
    # and the stored bricks are those holding a surface voxel of the cleared planes
    keys, bt, bc = st.sorted()
    b = g >> 3
    surf = (c0[:, 3] != 0) & (t0 != mo.DIVISOR)
    assert np.array_equal(keys, np.unique(mv.brick_key(b[surf, 0], b[surf, 1], b[surf, 2])).astype(np.uint64))
