"""The marching-cubes case table (tools/gen_mc_table.py -> kintinuous_b200/csrc/kt_mc_table.h) and the numpy restatement of the mesher
(oracle/mesh_oracle.py) on analytic surfaces.  CPU only."""
import importlib.util
import os
import sys

import numpy as np
import pytest

from conftest import ROOT

sys.path.insert(0, ROOT)
from oracle import mesh_oracle as mo  # noqa: E402


def _gen():
    spec = importlib.util.spec_from_file_location("gen_mc_table", os.path.join(ROOT, "tools", "gen_mc_table.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_generator_reproduces_header():
    g = _gen()
    with open(os.path.join(ROOT, "kintinuous_b200", "csrc", "kt_mc_table.h")) as f:
        assert f.read() == g.render_header(g.build_table())


def _boundary(tris):
    """directed edges (p, q) of the triangle fan that no triangle runs the other way: the outline of each loop"""
    d = set()
    for t in tris:
        for k in range(3):
            d.add((t[k], t[(k + 1) % 3]))
    return {e for e in d if (e[1], e[0]) not in d}


def _face_edges(g, f, s):
    return {e for e in range(12) if e >> 2 != f and all((c >> f) & 1 == s for c in g.edge_corners(e))}


def _table_face_segments(g, tris, f, s):
    fe = _face_edges(g, f, s)
    return {e for e in _boundary(tris) if e[0] in fe and e[1] in fe}


def test_loops_are_closed():
    g = _gen()
    cnt, tab = mo.load_table()
    for c in range(256):
        tris = [tuple(int(v) for v in tab[c, 3 * k:3 * k + 3]) for k in range(cnt[c])]
        assert tris == g.case_triangles(c)
        b = _boundary(tris)
        heads = sorted(e[1] for e in b); tails = sorted(e[0] for e in b)
        assert heads == tails                                   # every outline vertex is entered once and left once: closed loops
        crossing = {e for e in range(12) if len({(c >> k) & 1 for k in g.edge_corners(e)}) == 2}
        assert set(heads) == crossing and len(heads) == len(crossing)
        # the outline is exactly the segments on the six faces
        segs = set()
        for f, s, cyc in g.faces():
            segs |= set(g.face_segments(c, f, s, cyc))
        assert b == segs, c


def test_neighbouring_cells_agree_on_shared_faces():
    """For every pair of cases that agree on a shared face, in each axis, the two cells put the same segments on it (in opposite
    directions), read from the table's triangles."""
    g = _gen()
    cnt, tab = mo.load_table()
    tris = [[tuple(int(v) for v in tab[c, 3 * k:3 * k + 3]) for k in range(cnt[c])] for c in range(256)]
    pairs = 0
    for f in range(3):
        hi = [c for c in range(8) if (c >> f) & 1]                  # corners of cell A on its upper face ...
        lo = [c & ~(1 << f) for c in hi]                            # ... are the corners of cell B on its lower face
        def edge_map(e):                                            # A's edge on the face -> the same edge of B
            c0, c1 = g.edge_corners(e)
            return g.edge_of(c0 & ~(1 << f), c1 & ~(1 << f))
        segA = [_table_face_segments(g, tris[a], f, 1) for a in range(256)]
        segB = [_table_face_segments(g, tris[b], f, 0) for b in range(256)]
        for a in range(256):
            for b in range(256):
                if any(((a >> ch) & 1) != ((b >> cl) & 1) for ch, cl in zip(hi, lo)):
                    continue
                pairs += 1
                mapped = {(edge_map(q), edge_map(p)) for p, q in segA[a]}      # reversed direction
                assert mapped == segB[b], (f, a, b)
    assert pairs == 3 * 256 * 16


V = 128
C0 = np.array([64.3, 63.8, 64.1])


def _grid():
    z, y, x = np.meshgrid(np.arange(V), np.arange(V), np.arange(V), indexing="ij")
    return np.stack([x, y, z], -1) + 0.5                           # voxel centres, voxel units, [z, y, x, 3]


def _sphere(p, c=C0, r=40.0):
    d = p - c
    n = np.linalg.norm(d, axis=-1)
    return n - r, d / np.maximum(n, 1e-12)[..., None]


def _torus(p, R=32.0, r=12.0):
    d = p - C0
    q = np.hypot(d[..., 0], d[..., 1])
    s = np.stack([q - R, d[..., 2]], -1)
    dist = np.linalg.norm(s, axis=-1) - r
    u = s / np.maximum(np.linalg.norm(s, axis=-1), 1e-12)[..., None]
    radial = np.stack([d[..., 0], d[..., 1]], -1) / np.maximum(q, 1e-12)[..., None]
    n = np.concatenate([u[..., :1] * radial, u[..., 1:]], -1)
    return dist, n


AXIS2 = np.array([1.0, 1.0, 0.35]) / np.linalg.norm([1.0, 1.0, 0.35])


def _two_spheres(p, r=24.0, gap=0.8):
    ca, cb = C0 - AXIS2 * (r + gap / 2), C0 + AXIS2 * (r + gap / 2)
    da, na = _sphere(p, ca, r)
    db, nb = _sphere(p, cb, r)
    first = (da <= db)[..., None]
    return np.minimum(da, db), np.where(first, na, nb)


SHAPES = {"sphere": (_sphere, 2), "torus": (_torus, 0), "two_spheres": (_two_spheres, 4)}


def analytic_volume(name):
    fn, _ = SHAPES[name]
    d, _ = fn(_grid())
    rng = np.random.default_rng(7)
    col = rng.integers(0, 256, size=(V, V, V, 4), dtype=np.uint8)
    return mo.sdf_volume(d, 4.0, 20, col)


def mesh_stats(verts, tris):
    e = np.concatenate([tris[:, [0, 1]], tris[:, [1, 2]], tris[:, [2, 0]]])
    und = np.sort(e, 1)
    keys, counts = np.unique(und[:, 0].astype(np.int64) * (1 << 32) + und[:, 1], return_counts=True)
    dkeys = np.unique(e[:, 0].astype(np.int64) * (1 << 32) + e[:, 1])
    return dict(V=len(verts), E=len(keys), F=len(tris), edge_uses=counts, directed_unique=len(dkeys), directed=len(e))


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_oracle_on_analytic_surfaces(name):
    fn, chi = SHAPES[name]
    tsdf, col = analytic_volume(name)
    size = float(V)                                                # 1 m per voxel: positions are in voxels
    v, t = mo.mesh(tsdf, col, V, size, (0, 0, 0), (0, 0, 0), (0, V, 0, V, 0, V), 8)
    assert len(t) > 1000
    st = mesh_stats(v, t)
    assert (st["edge_uses"] == 2).all()                            # closed 2-manifold ...
    assert st["directed_unique"] == st["directed"]                 # ... consistently oriented: each edge once per direction
    assert st["V"] - st["E"] + st["F"] == chi, (name, st["V"] - st["E"] + st["F"])
    assert len(np.unique(t)) == len(v)                             # no unreferenced vertex
    p = np.stack([v["x"], v["y"], v["z"]], -1).astype(np.float64) + size / 2        # back to volume coordinates
    d, _ = fn(p)
    print(f"{name}: {len(v)} vertices, {len(t)} triangles, chi {chi}, max |sdf| at vertices {np.abs(d).max():.4f} voxel")
    if name == "two_spheres":
        # min(d_a, d_b) has a crease in the gap: an edge whose ends are nearest to different spheres interpolates across it.  The
        # 0.05-voxel bound holds wherever the other sphere is more than 1.5 voxels away; in the gap the crease costs up to ~0.1 voxel.
        ra, rb = _sphere(p, C0 - AXIS2 * 24.4, 24.0)[0], _sphere(p, C0 + AXIS2 * 24.4, 24.0)[0]
        far = np.maximum(ra, rb) > 1.5
        assert far.mean() > 0.99 and np.abs(d[far]).max() <= 0.05 and np.abs(d).max() <= 0.15
    else:
        assert np.abs(d).max() <= 0.05
    a, b, c = p[t[:, 0]], p[t[:, 1]], p[t[:, 2]]
    n = np.cross(b - a, c - a)
    area = np.linalg.norm(n, axis=1)
    keep = area > 1e-4                                             # slivers (a vertex next to a corner) have no meaningful normal
    cen = (a + b + c) / 3
    if name == "two_spheres":                                      # which sphere a centroid in the gap belongs to is ambiguous
        keep &= np.maximum(_sphere(cen, C0 - AXIS2 * 24.4, 24.0)[0], _sphere(cen, C0 + AXIS2 * 24.4, 24.0)[0]) > 1.5
    _, na = fn(cen)
    cosang = (n[keep] * na[keep]).sum(1) / area[keep]
    print(f"{name}: triangle normal vs analytic: min cos {cosang.min():.3f}, 1 % quantile {np.quantile(cosang, 0.01):.3f}")
    assert (cosang > 0).all()
    vn = np.stack([v["nx"], v["ny"], v["nz"]], -1).astype(np.float64)
    _, nv = fn(p)
    assert np.median((vn * nv).sum(1)) > 0.99
    if name == "two_spheres":                                      # the case this volume is for: ambiguous faces are met
        assert _ambiguous_faces(tsdf) > 0


def _ambiguous_faces(tsdf):
    ins = tsdf < 0
    n = 0
    for ax in range(3):
        a = np.moveaxis(ins, ax, 0)
        c00, c10, c01, c11 = a[:, :-1, :-1], a[:, 1:, :-1], a[:, :-1, 1:], a[:, 1:, 1:]
        n += int(((c00 == c11) & (c10 == c01) & (c00 != c10)).sum())
    return n
