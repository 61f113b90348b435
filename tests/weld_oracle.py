"""numpy restatement of the keyed marching cubes (kt_op_mesh_volume_keyed) and of the mesh weld (kt_op_weld_meshes, kt_weld.cu),
test-only, on top of oracle/mesh_oracle.py.

keyed() returns mesh_oracle.mesh's vertices and triangles with their global keys: each vertex's edge (gx, gy, gz, axis) is
mesh_oracle's owner plus real_wrap, and each triangle's cell (gx, gy, gz, 0) is the lower corner of the meshed cell it comes from (cells
in logical order, each repeated by its case's triangle count, which is the order mesh_oracle emits triangles in) plus real_wrap."""
from __future__ import annotations

import numpy as np

from oracle import mesh_oracle as mo

KEY_LIMIT = 1 << 62


def triangle_cells(tsdf, color, V, wrap, box, weight_cull=8, table=None):
    """Lower corner (x, y, z, 0) in logical coordinates of the cell of every triangle mesh_oracle.mesh emits, in its order."""
    cnt, _ = table if table is not None else mo.load_table()
    minX, maxX, minY, maxY, minZ, maxZ = box
    if maxX <= minX or maxY <= minY or maxZ <= minZ:
        return np.zeros((0, 4), np.int64)
    T = mo.logical(tsdf, wrap, V).astype(np.int32)
    W = mo.logical(color, wrap, V)[..., 3].astype(np.int32)
    valid = (W != 0) & (T != mo.DIVISOR) & (W >= weight_cull)
    inside = T < 0
    case = np.zeros((V - 1, V - 1, V - 1), np.int64)
    allv = np.ones((V - 1, V - 1, V - 1), bool)
    for k in range(8):
        dx, dy, dz = k & 1, (k >> 1) & 1, k >> 2
        sl = (slice(dz, dz + V - 1), slice(dy, dy + V - 1), slice(dx, dx + V - 1))
        allv &= valid[sl]
        case |= inside[sl].astype(np.int64) << k
    meshed = allv & (case != 0) & (case != 255)
    inbox = np.zeros_like(meshed)
    inbox[minZ:min(maxZ, V - 1), minY:min(maxY, V - 1), minX:min(maxX, V - 1)] = True
    meshed &= inbox
    cz, cy, cx = np.nonzero(meshed)                                     # C order: z, then y, then x fastest
    nt = cnt[case[cz, cy, cx]]
    return np.repeat(np.stack([cx, cy, cz, np.zeros_like(cx)], -1), nt, axis=0).astype(np.int64).reshape(-1, 4)


def keyed(tsdf, color, V, volume_size, wrap, real_wrap, box, weight_cull=8, table=None):
    """(vertices, triangles uint32 [m, 3], edges int64 [n, 4], cells int64 [m, 4]) with global keys, as kt_op_mesh_volume_keyed."""
    table = table if table is not None else mo.load_table()
    v, t, own = mo.mesh(tsdf, color, V, volume_size, wrap, real_wrap, box, weight_cull, table, return_owners=True)
    cells = triangle_cells(tsdf, color, V, wrap, box, weight_cull, table)
    assert len(cells) == len(t), "the cell enumeration disagrees with mesh_oracle.mesh"
    rw = np.asarray(real_wrap, np.int64)
    e = own.astype(np.int64).copy(); e[:, :3] += rw
    c = cells.copy(); c[:, :3] += rw
    return v, t, e, c


def weld(meshes):
    """kt_op_weld_meshes restated: meshes = [(vertices MESH_VERTEX_DTYPE [n], triangles uint32 [m, 3] local to the mesh, edges int [n, 4]
    global (gx, gy, gz, axis), cells int [m, 4] global (gx, gy, gz, 0))], in order.  Returns (vertices, triangles uint32 [k, 3], edges
    int64 [.., 4], cells int64 [k, 4], stats dict).
      * cell winner: each cell keeps the triangles of the highest-numbered mesh with triangles there;
      * vertex weld: the vertices kept triangles use; per global edge the highest-numbered mesh's vertex;
      * order: vertices by (gz, gy, gx, axis), triangles by cell (gz, gy, gx) then the winner's order.
    ValueError for an index outside its mesh, an axis outside 0..2, no mesh, or 3 x the voxels of the lattice box the keys span
    beyond 2^62 (the device's 64-bit keys)."""
    if not meshes:
        raise ValueError("no mesh")
    V = [np.asarray(m[0]) for m in meshes]
    T = [np.asarray(m[1], np.int64).reshape(-1, 3) for m in meshes]
    E = [np.asarray(m[2], np.int64).reshape(-1, 4) for m in meshes]
    Cc = [np.asarray(m[3], np.int64).reshape(-1, 4) for m in meshes]
    nvs = np.array([len(v) for v in V], np.int64); nts = np.array([len(t) for t in T], np.int64)
    voff = np.concatenate([[0], np.cumsum(nvs)])
    verts = np.concatenate(V)
    tris = np.concatenate(T); edges = np.concatenate(E); cells = np.concatenate(Cc)
    tmesh = np.repeat(np.arange(len(meshes)), nts)
    stats = dict(input_verts=int(voff[-1]), input_tris=int(nts.sum()), output_verts=0, output_tris=0, repeated_cells=0, dropped_triangles=0,
                 merged_vertices=0, meshes=len(meshes))
    if len(tris) == 0:
        return np.zeros(0, mo.MESH_VERTEX_DTYPE), np.zeros((0, 3), np.uint32), np.zeros((0, 4), np.int64), np.zeros((0, 4), np.int64), stats
    if ((tris < 0) | (tris >= nvs[tmesh][:, None])).any():
        raise ValueError("a triangle index is outside its mesh")
    if ((edges[:, 3] < 0) | (edges[:, 3] > 2)).any():
        raise ValueError("an edge axis is outside 0..2")
    allc = np.concatenate([edges[:, :3], cells[:, :3]])
    lo, hi = allc.min(0), allc.max(0)
    ext = [int(h) - int(l) + 1 for l, h in zip(lo, hi)]
    if 3 * ext[0] * ext[1] * ext[2] > KEY_LIMIT:
        raise ValueError("keys beyond 2^62")
    ckey = lambda c: (c[:, 0] - lo[0]) + ext[0] * ((c[:, 1] - lo[1]) + ext[1] * (c[:, 2] - lo[2]))   # noqa: E731
    tk = ckey(cells)
    order = np.lexsort((np.arange(len(tk)), tk))                         # by cell, then input order (mesh, then the mesh's order)
    tk_s, tm_s = tk[order], tmesh[order]
    ucell, first, inv = np.unique(tk_s, return_index=True, return_inverse=True)
    win = np.full(len(ucell), -1); np.maximum.at(win, inv, tm_s)
    keep = tm_s == win[inv]
    stats["repeated_cells"] = int((tm_s[first] != win).sum())
    kept = order[keep]
    gidx = tris[kept] + voff[tmesh[kept]][:, None]                      # global vertex indices of the kept triangles
    used = np.zeros(len(verts), bool); used[gidx.ravel()] = True
    ekey = 3 * ckey(edges) + edges[:, 3]
    ui = np.nonzero(used)[0]
    vorder = ui[np.lexsort((ui, ekey[ui]))]                             # by edge key, then input order (mesh)
    ek_s = ekey[vorder]
    last = np.ones(len(vorder), bool); last[:-1] = ek_s[1:] != ek_s[:-1]
    rep_idx = vorder[last]; ukeys = ek_s[last]
    out_t = np.searchsorted(ukeys, ekey[gidx]).astype(np.uint32)
    stats.update(output_verts=len(rep_idx), output_tris=len(kept), dropped_triangles=int(len(tris) - len(kept)),
                 merged_vertices=int(len(ui) - len(rep_idx)))
    return verts[rep_idx].copy(), out_t, edges[rep_idx].copy(), cells[kept].copy(), stats
