"""numpy restatement of kt_op_mesh_volume (kintinuous_b200/csrc/kt_mesh.cu), test-only.

It reads the committed case table (kintinuous_b200/csrc/kt_mc_table.h) and restates the contract: corner validity, meshed cells,
vertex ownership and order, triangles in cell then table order, normals in float64.  Positions follow extract_kernel's interp in
float32, in its order, but numpy neither fuses the multiply-add nor uses the kernel's approximate reciprocal, so they match the
kernel to a tolerance, not bit for bit.

Volumes are in the reference layout: tsdf int16 [V, V, V] and colour uint8 [V, V, V, 4] indexed [z, y, x] in STORAGE order; logical
voxel (x, y, z) is stored at ((x + wrap.x) mod V, ...)."""
from __future__ import annotations

import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "kintinuous_b200", "csrc", "kt_mc_table.h")
DIVISOR = 32767


def load_table(path=HEADER):
    """(tri_count uint8 [256], tris uint8 [256, 3 * max]) parsed from the header."""
    txt = open(path).read()
    mt = int(re.search(r"#define KT_MC_MAX_TRIS (\d+)", txt).group(1))
    body = txt[txt.index("kt_mc_tri_count[256] = {"):]
    cnt = np.array([int(v) for v in re.findall(r"\d+", body[body.index("{") + 1:body.index("}")])], np.int64)
    rest = body[body.index("kt_mc_tris[256]"):]
    rows = re.findall(r"\{([\d, ]+)\}", rest)
    tris = np.array([[int(v) for v in r.split(",")] for r in rows], np.int64)
    assert cnt.shape == (256,) and tris.shape == (256, 3 * mt)
    return cnt, tris


# edge e = 4 a + j: axis and the offset of its lower corner (kt_mc_table.h)
EDGE_AXIS = np.array([e >> 2 for e in range(12)])
EDGE_OFF = np.array([[0, j & 1, j >> 1] if a == 0 else [j & 1, 0, j >> 1] if a == 1 else [j & 1, j >> 1, 0]
                     for a, j in ((e >> 2, e & 3) for e in range(12))])     # (dx, dy, dz)
MESH_VERTEX_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4"),
                              ("r", "u1"), ("g", "u1"), ("b", "u1"), ("a", "u1"), ("_pad", "<u4")])


def logical(arr, wrap, V):
    """storage -> logical order ([z, y, x]): logical (x, y, z) is storage ((x + wx) mod V, ...)"""
    w = [int(v) % V for v in wrap]
    return np.roll(arr, shift=(-w[2], -w[1], -w[0]), axis=(0, 1, 2))


def mesh(tsdf, color, V, volume_size, wrap, real_wrap, box, weight_cull=8, table=None, return_owners=False):
    """Returns (vertices MESH_VERTEX_DTYPE [n], triangles uint32 [m, 3]) as kt_op_mesh_volume defines them; with return_owners also
    each vertex's edge as (x, y, z, axis) of its lower voxel in logical coordinates."""
    cnt, tab = table if table is not None else load_table()
    minX, maxX, minY, maxY, minZ, maxZ = box
    vs = np.broadcast_to(np.asarray(volume_size, np.float32), (3,))
    cell = (vs / np.float32(V)).astype(np.float32)                     # (x, y, z)
    T = logical(tsdf, wrap, V).astype(np.int32)
    Cl = logical(color, wrap, V)
    W = Cl[..., 3].astype(np.int32)
    valid = (W != 0) & (T != DIVISOR) & (W >= weight_cull)            # F = raw / 32767 == 1 only for raw == 32767
    inside = T < 0
    empty = (np.zeros(0, MESH_VERTEX_DTYPE), np.zeros((0, 3), np.uint32)) + ((np.zeros((0, 4), np.int64),) if return_owners else ())
    if maxX <= minX or maxY <= minY or maxZ <= minZ:
        return empty

    # meshed cells, indexed [z, y, x] over the whole volume (lower corners)
    meshed = np.zeros((V, V, V), bool)
    case = np.zeros((V - 1, V - 1, V - 1), np.int64)
    allv = np.ones((V - 1, V - 1, V - 1), bool)
    for k in range(8):
        dx, dy, dz = k & 1, (k >> 1) & 1, k >> 2
        sl = (slice(dz, dz + V - 1), slice(dy, dy + V - 1), slice(dx, dx + V - 1))
        allv &= valid[sl]
        case |= inside[sl].astype(np.int64) << k
    m = allv & (case != 0) & (case != 255)
    inbox = np.zeros_like(m)
    inbox[minZ:min(maxZ, V - 1), minY:min(maxY, V - 1), minX:min(maxX, V - 1)] = True
    meshed[:V - 1, :V - 1, :V - 1] = m & inbox

    # owner grid [min, min(max + 1, V)) per axis
    ex1, ey1, ez1 = min(maxX + 1, V), min(maxY + 1, V), min(maxZ + 1, V)
    ex, ey = ex1 - minX, ey1 - minY
    Mp = np.pad(meshed, ((1, 0), (1, 0), (1, 0)))                      # Mp[z + 1, y + 1, x + 1] = meshed[z, y, x]; -1 -> False
    keys, owners = [], []
    zz, yy, xx = np.meshgrid(np.arange(minZ, ez1), np.arange(minY, ey1), np.arange(minX, ex1), indexing="ij")
    for a in range(3):
        d = [0, 0, 0]; d[a] = 1                                      # (dx, dy, dz)
        nx_, ny_, nz_ = xx + d[0], yy + d[1], zz + d[2]
        ok = (nx_ < V) & (ny_ < V) & (nz_ < V)
        nxc, nyc, nzc = np.minimum(nx_, V - 1), np.minimum(ny_, V - 1), np.minimum(nz_, V - 1)
        cross = ok & valid[zz, yy, xx] & valid[nzc, nyc, nxc] & (inside[zz, yy, xx] != inside[nzc, nyc, nxc])
        used = np.zeros_like(cross)
        others = [b for b in range(3) if b != a]
        for s0 in (0, 1):
            for s1 in (0, 1):
                o = [0, 0, 0]; o[others[0]] = s0; o[others[1]] = s1
                used |= Mp[zz - o[2] + 1, yy - o[1] + 1, xx - o[0] + 1]
        sel = cross & used
        lin = (xx - minX) + ex * ((yy - minY) + ey * (zz - minZ))
        keys.append(3 * lin[sel].astype(np.int64) + a)
        owners.append(np.stack([xx[sel], yy[sel], zz[sel], np.full(int(sel.sum()), a)], -1))
    keys = np.concatenate(keys); owners = np.concatenate(owners)
    order = np.argsort(keys, kind="stable")
    keys = keys[order]; owners = owners[order]
    n = len(keys)
    if n == 0:
        return empty

    x, y, z, a = owners.T
    d = np.zeros((n, 3), np.int64); d[np.arange(n), a] = 1
    x1, y1, z1 = x + d[:, 0], y + d[:, 1], z + d[:, 2]
    r0, r1 = T[z, y, x], T[z1, y1, x1]
    # position: extract_kernel's point, float32
    F = r0.astype(np.float32) / np.float32(DIVISOR); Fn = r1.astype(np.float32) / np.float32(DIVISOR)
    Vc = np.stack([(x.astype(np.float32) + np.float32(0.5)) * cell[0], (y.astype(np.float32) + np.float32(0.5)) * cell[1],
                   (z.astype(np.float32) + np.float32(0.5)) * cell[2]], -1).astype(np.float32)
    d_inv = (np.float32(1) / (np.abs(F) + np.abs(Fn))).astype(np.float32)
    va = Vc[np.arange(n), a]; vn = (va + cell[a]).astype(np.float32)
    Vc[np.arange(n), a] = ((va * np.abs(Fn) + np.abs(F) * vn) * d_inv).astype(np.float32)
    rw = np.asarray(real_wrap, np.int64)
    pos = (Vc + (rw.astype(np.float32) * cell) - ((cell * np.float32(V)) / np.float32(2))).astype(np.float32)

    # normal: gradient (raw units per metre) at both ends, blended by the position's weights, float64
    def grad(px, py, pz):
        g = np.zeros((len(px), 3))
        c = np.stack([px, py, pz], -1)
        r = T[pz, py, px].astype(np.float64)
        for b in range(3):
            e = np.zeros(3, np.int64); e[b] = 1
            cm, cp = c - e, c + e
            okm = (cm[:, b] >= 0); okp = (cp[:, b] < V)
            cmc = np.clip(cm, 0, V - 1); cpc = np.clip(cp, 0, V - 1)
            okm &= valid[cmc[:, 2], cmc[:, 1], cmc[:, 0]]; okp &= valid[cpc[:, 2], cpc[:, 1], cpc[:, 0]]
            rm = T[cmc[:, 2], cmc[:, 1], cmc[:, 0]].astype(np.float64); rp = T[cpc[:, 2], cpc[:, 1], cpc[:, 0]].astype(np.float64)
            h = float(cell[b])
            g[:, b] = np.where(okm & okp, (rp - rm) / (2 * h), np.where(okp, (rp - r) / h, np.where(okm, (r - rm) / h, 0.0)))
        return g
    a0, a1 = np.abs(r0.astype(np.float64)), np.abs(r1.astype(np.float64))
    w0 = (a1 / (a0 + a1))[:, None]; w1 = (a0 / (a0 + a1))[:, None]
    nrm = w0 * grad(x, y, z) + w1 * grad(x1, y1, z1)
    ln = np.linalg.norm(nrm, axis=1)
    nrm = np.where(ln[:, None] > 0, nrm / np.where(ln > 0, ln, 1)[:, None], 0.0)

    lower = np.abs(r0) <= np.abs(r1)
    cx, cy, cz = np.where(lower, x, x1), np.where(lower, y, y1), np.where(lower, z, z1)
    col = Cl[cz, cy, cx]
    v = np.zeros(n, MESH_VERTEX_DTYPE)
    v["x"], v["y"], v["z"] = pos[:, 0], pos[:, 1], pos[:, 2]
    v["nx"], v["ny"], v["nz"] = nrm[:, 0], nrm[:, 1], nrm[:, 2]
    v["r"], v["g"], v["b"], v["a"] = col[:, 2], col[:, 1], col[:, 0], col[:, 3]

    # triangles: meshed cells in logical order, then table order
    cz_, cy_, cx_ = np.nonzero(meshed)                                   # C order: z, then y, then x fastest
    cc = case[cz_, cy_, cx_]
    nt = cnt[cc]
    cell_id = np.repeat(np.arange(len(cc)), nt)
    slot = np.arange(int(nt.sum())) - np.repeat(np.cumsum(nt) - nt, nt)
    edges = np.stack([tab[cc[cell_id], 3 * slot + k] for k in range(3)], -1)       # [m, 3]
    lin = (cx_ - minX) + ex * ((cy_ - minY) + ey * (cz_ - minZ))
    off = EDGE_OFF[edges]                                                        # [m, 3, 3]
    olin = lin[cell_id][:, None] + off[..., 0] + ex * (off[..., 1] + ey * off[..., 2])
    tkeys = 3 * olin.astype(np.int64) + EDGE_AXIS[edges]
    idx = np.searchsorted(keys, tkeys)
    assert (idx < n).all() and (keys[np.minimum(idx, n - 1)] == tkeys).all(), "a triangle references an edge without a vertex"
    return (v, idx.astype(np.uint32)) + ((owners,) if return_owners else ())


def sdf_volume(sdf_vox, trunc_vox=4.0, weight=20, color=None):
    """(tsdf int16, colour uint8 [.., 4]) of an SDF sampled at the voxel centres (in voxels), truncated like the integration (raw =
    clamp(d / trunc, -1, 1) * 32767, truncated towards zero), every voxel observed with `weight`."""
    f = np.clip(sdf_vox / trunc_vox, -1.0, 1.0)
    tsdf = np.trunc(f * DIVISOR).astype(np.int16)
    c = np.zeros(tsdf.shape + (4,), np.uint8) if color is None else color.copy()
    c[..., 3] = weight
    return tsdf, c
