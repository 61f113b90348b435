"""weld_oracle.weld, the numpy restatement of kt_op_weld_meshes (kt_weld.cu), on the CPU: welding the keyed marching-cubes meshes of
two overlapping boxes of one volume gives exactly the mesh of the union box, welding one mesh changes nothing, the latest mesh wins a
cell both meshed, and keys beyond 2^62 are refused."""
import numpy as np
import pytest

from oracle import mesh_oracle as mo
from weld_oracle import keyed as keyed_mesh, weld

V = 40


def _volume(seed=1):
    z, y, x = np.meshgrid(*[np.arange(V)] * 3, indexing="ij")
    d = np.sqrt((x - 17.3) ** 2 + (y - 21.1) ** 2 + (z - 19.7) ** 2) - 11.2 + 0.8 * np.sin(x * 0.7) * np.cos(y * 0.5)
    rng = np.random.default_rng(seed)
    col = rng.integers(0, 256, (V, V, V, 4), dtype=np.uint8)
    return mo.sdf_volume(d.astype(np.float32), color=col)


def _store(t, c, wrap):
    w = [int(v) % V for v in wrap]
    return np.roll(t, (w[2], w[1], w[0]), (0, 1, 2)), np.roll(c, (w[2], w[1], w[0]), (0, 1, 2))


TABLE = mo.load_table()


def keyed(t, c, wrap, rw, box):
    """(vertices, triangles, global edges, global cells) of one box"""
    return keyed_mesh(t, c, V, 6.0, wrap, rw, box, 8, TABLE)


def _same(got, want, label):
    gv, gt, ge, gc = got[:4]; wv, wt, we, wc = want[:4]
    assert gv.tobytes() == wv.tobytes(), label                          # positions, normals, colours bit for bit
    assert np.array_equal(gt, wt) and np.array_equal(ge, we) and np.array_equal(gc, wc), label


SPLITS = [((0, 20, 0, V, 0, V), (16, V, 0, V, 0, V)),
          ((0, V, 0, 25, 0, V), (0, V, 22, V, 0, V)),
          ((0, V, 0, V, 0, 18), (0, V, 0, V, 14, V - 1))]               # z: the ZMinus slab ends at V - 1


@pytest.mark.parametrize("wrap,rw", [((7, 3, 11), (-5, 40, 2)), ((0, 29, 5), (12, -33, -70))])
@pytest.mark.parametrize("split", range(len(SPLITS)))
def test_weld_of_overlapping_boxes_is_the_union_box(wrap, rw, split):
    t, c = _store(*_volume(), wrap)
    A, B = SPLITS[split]
    U = tuple(min(A[i], B[i]) if i % 2 == 0 else max(A[i], B[i]) for i in range(6))
    ma, mb, mu = keyed(t, c, wrap, rw, A), keyed(t, c, wrap, rw, B), keyed(t, c, wrap, rw, U)
    assert len(mu[1]) > 1000
    for order in ((ma, mb), (mb, ma)):                                  # either box may be the later one
        got = weld(list(order))
        _same(got, mu, (split, wrap))
        st = got[4]
        assert st["repeated_cells"] > 0 and st["dropped_triangles"] == len(ma[1]) + len(mb[1]) - len(mu[1])
        assert st["merged_vertices"] > 0 and st["output_verts"] == len(mu[0])


def test_welding_one_mesh_is_the_identity():
    t, c = _store(*_volume(), (3, 5, 7))
    m = keyed(t, c, (3, 5, 7), (1, -2, 3), (4, 33, 0, V, 2, 30))
    got = weld([m])
    _same(got, m, "one mesh")
    assert got[4]["repeated_cells"] == 0 and got[4]["merged_vertices"] == 0


def test_latest_mesh_wins_its_cells():
    t, c = _volume()
    A, B = (0, 22, 0, V, 0, V), (16, V, 0, V, 0, V)
    # B's volume: the surface moved by half a voxel in (and beyond) the overlap planes, as if later frames had refined it
    z, y, x = np.meshgrid(*[np.arange(V)] * 3, indexing="ij")
    d = np.sqrt((x - 17.3) ** 2 + (y - 21.1) ** 2 + (z - 19.7) ** 2) - 11.7 + 0.8 * np.sin(x * 0.7) * np.cos(y * 0.5)
    t2, _ = mo.sdf_volume(d.astype(np.float32))
    t2 = np.where(x >= 16, t2, t)
    ma, mb = keyed(t, c, (0, 0, 0), (0, 0, 0), A), keyed(t2, c, (0, 0, 0), (0, 0, 0), B)
    wv, wt, we, wc, st = weld([ma, mb])

    def tri_set(m):
        v, tr, e, k = m[:4]
        return {(tuple(k[i][:3]),) + tuple(tuple(e[j]) for j in tr[i]) for i in range(len(tr))}
    cells_b = {tuple(k[:3]) for k in mb[3]}
    only_a = {tuple(k[:3]) for k in ma[3]} - cells_b
    want = {x for x in tri_set(ma) if x[0] in only_a} | tri_set(mb)
    assert tri_set((wv, wt, we, wc)) == want
    overlap_only_a = [k for k in only_a if k[0] >= 16]
    assert overlap_only_a, "the moved surface leaves cells that only the earlier mesh has"
    assert st["repeated_cells"] > 0 and st["dropped_triangles"] > 0
    # representatives: B's vertex wherever B has one on the edge, else A's
    vb = {tuple(e): v.tobytes() for e, v in zip(mb[2], mb[0])}
    va = {tuple(e): v.tobytes() for e, v in zip(ma[2], ma[0])}
    for e, v in zip(we, wv):
        assert v.tobytes() == vb.get(tuple(e), va.get(tuple(e)))
    assert any(tuple(e) in va and tuple(e) in vb and va[tuple(e)] != vb[tuple(e)] for e in we)


def test_key_range_is_refused():
    v = np.zeros(3, mo.MESH_VERTEX_DTYPE)
    e = np.array([[-2 ** 30, 0, 0, 0], [2 ** 30, 2 ** 30, 0, 1], [0, -2 ** 30, 2 ** 30, 2]])
    m = (v, np.array([[0, 1, 2]], np.uint32), e, np.array([[0, 0, 0, 0]]))
    with pytest.raises(ValueError, match="2\\^62"):
        weld([m])
    small = e // 2 ** 20
    assert weld([(v, m[1], small, m[3])])[4]["output_tris"] == 1
    with pytest.raises(ValueError, match="outside its mesh"):
        weld([(v, np.array([[0, 1, 3]], np.uint32), small, m[3])])


def test_every_triangle_uses_edges_of_its_cell():
    """the cells (enumerated from the volume) and the triangles' edges (mesh_oracle) describe the same cubes"""
    wrap, rw = (5, 0, 33), (-3, 8, 21)
    t, c = _store(*_volume(), wrap)
    v, tr, e, k = keyed(t, c, wrap, rw, (3, 37, 0, V, 6, V - 1))
    assert len(tr) > 1000
    off = e[tr.astype(np.int64)][..., :3] - k[:, None, :3]              # [m, 3 vertices, 3 axes]
    axis = e[tr.astype(np.int64)][..., 3]
    assert ((off == 0) | (off == 1)).all()
    assert (np.take_along_axis(off, axis[..., None], -1) == 0).all()    # an edge lies along its axis from the cell's corner plane
