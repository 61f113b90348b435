"""numpy restatement of the map volume (kintinuous_b200/csrc/kt_mapvol.cu), test-only, on top of oracle/mesh_oracle.py.

Store: a dict brick key -> (tsdf int16 [8, 8, 8], colour uint8 [8, 8, 8, 4]) indexed [z, y, x] inside the brick.  Before each clear, the
surface voxels of the cleared planes (W != 0, raw != 32767) create their bricks and every cleared voxel with W != 0 overwrites its value
in a brick that exists; a clear whose new bricks would take the store past its capacity creates none of them.  The map field S is the
store where the live volume has W = 0, else the live volume; global voxel = logical voxel + the real voxel wrap.  The map mesh is
mesh_oracle.mesh over S with no border, vertex positions computed from the global voxel with real wrap 0."""
from __future__ import annotations

import numpy as np

from oracle import mesh_oracle as mo

BIAS = 1 << 20


def brick_key(bx, by, bz):
    return ((np.asarray(bz, np.int64) + BIAS) << 42) | ((np.asarray(by, np.int64) + BIAS) << 21) | (np.asarray(bx, np.int64) + BIAS)


def key_brick(k):
    k = np.asarray(k, np.int64)
    return (k & 0x1FFFFF) - BIAS, (k >> 21 & 0x1FFFFF) - BIAS, (k >> 42) - BIAS


class Store:
    def __init__(self, capacity=None):
        self.bricks = {}
        self.capacity = capacity
        self.full = False

    def clear(self, g, tsdf, color):
        """Keep the cleared voxels: g int [n, 3] global (x, y, z), tsdf int16 [n], colour uint8 [n, 4]."""
        g = np.asarray(g, np.int64)
        W = color[:, 3]
        obs = W != 0
        b = g >> 3
        keys = brick_key(b[:, 0], b[:, 1], b[:, 2])
        new = [int(k) for k in np.unique(keys[obs & (tsdf != mo.DIVISOR)]) if int(k) not in self.bricks]
        if self.capacity is not None and len(self.bricks) + len(new) > self.capacity:
            self.full = True
        else:
            for k in new:
                self.bricks[k] = (np.zeros((8, 8, 8), np.int16), np.zeros((8, 8, 8, 4), np.uint8))
        sel = np.nonzero(obs)[0]
        uk, inv = np.unique(keys[sel], return_inverse=True)
        for j, k in enumerate(uk):
            if int(k) not in self.bricks:
                continue
            idx = sel[inv == j]
            l = g[idx] & 7
            t, c = self.bricks[int(k)]
            t[l[:, 2], l[:, 1], l[:, 0]] = tsdf[idx]
            c[l[:, 2], l[:, 1], l[:, 0]] = color[idx]

    def sorted(self):
        """(keys uint64 [n], tsdf [n, 8, 8, 8], colour [n, 8, 8, 8, 4]) in key order."""
        ks = sorted(self.bricks)
        if not ks:
            return np.zeros(0, np.uint64), np.zeros((0, 8, 8, 8), np.int16), np.zeros((0, 8, 8, 8, 4), np.uint8)
        return (np.array(ks, np.uint64), np.stack([self.bricks[k][0] for k in ks]), np.stack([self.bricks[k][1] for k in ks]))


def cleared_voxels(tsdf, color, V, axis, planes, wrap):
    """The voxels of storage planes `planes` along axis of a storage-order volume: (global [n, 3], tsdf [n], colour [n, 4], storage
    index tuple).  wrap: the signed voxel wrap at the clear."""
    s = [np.arange(V)] * 3
    s[axis] = np.asarray(planes, np.int64)
    sz, sy, sx = np.meshgrid(s[2], s[1], s[0], indexing="ij")
    sx, sy, sz = sx.ravel(), sy.ravel(), sz.ravel()
    st = np.stack([sx, sy, sz], -1)
    w = np.asarray(wrap, np.int64)
    g = (st - w % V) % V + w
    return g, tsdf[sz, sy, sx], color[sz, sy, sx], (sz, sy, sx)


def merged(store, tsdf, color, V, wrap):
    """S as a dense box: (tsdf, colour, origin) with origin = the global voxel of entry [0, 0, 0], a margin of 2 unobserved voxels all
    round (cubic, for mesh_oracle).  tsdf / colour: the live volume in storage order at the signed wrap."""
    w = np.asarray(wrap, np.int64)
    lo = [w.copy()]; hi = [w + V]
    for k in store.bricks:
        b = np.array(key_brick(k), np.int64)
        lo.append(8 * b); hi.append(8 * b + 8)
    lo = np.min(lo, 0) - 2; hi = np.max(hi, 0) + 2
    n = int((hi - lo).max())
    T = np.zeros((n, n, n), np.int16); C = np.zeros((n, n, n, 4), np.uint8)
    for k, (t, c) in store.bricks.items():
        o = 8 * np.array(key_brick(k), np.int64) - lo
        T[o[2]:o[2] + 8, o[1]:o[1] + 8, o[0]:o[0] + 8] = t
        C[o[2]:o[2] + 8, o[1]:o[1] + 8, o[0]:o[0] + 8] = c
    Tl = mo.logical(tsdf, w, V); Cl = mo.logical(color, w, V)
    o = w - lo
    sl = (slice(o[2], o[2] + V), slice(o[1], o[1] + V), slice(o[0], o[0] + V))
    live = Cl[..., 3] != 0
    T[sl] = np.where(live, Tl, T[sl]); C[sl] = np.where(live[..., None], Cl, C[sl])
    return T, C, lo


def box_bricks(T, C, origin):
    """The bricks of a dense box that hold an observed voxel, as sorted (keys, tsdf, colour); origin must be a multiple of 8 away from the
    brick lattice after padding, so the box is padded to whole bricks here."""
    o = np.asarray(origin, np.int64)
    b0 = o >> 3
    pad_lo = o - 8 * b0
    n = T.shape[0]
    m = [int(-(-(pad_lo[a] + n) // 8) * 8) for a in range(3)]
    Tp = np.zeros((m[2], m[1], m[0]), np.int16); Cp = np.zeros((m[2], m[1], m[0], 4), np.uint8)
    Tp[pad_lo[2]:pad_lo[2] + n, pad_lo[1]:pad_lo[1] + n, pad_lo[0]:pad_lo[0] + n] = T
    Cp[pad_lo[2]:pad_lo[2] + n, pad_lo[1]:pad_lo[1] + n, pad_lo[0]:pad_lo[0] + n] = C
    nb = [m[a] // 8 for a in range(3)]
    tb = Tp.reshape(nb[2], 8, nb[1], 8, nb[0], 8).transpose(0, 2, 4, 1, 3, 5).reshape(-1, 8, 8, 8)
    cb = Cp.reshape(nb[2], 8, nb[1], 8, nb[0], 8, 4).transpose(0, 2, 4, 1, 3, 5, 6).reshape(-1, 8, 8, 8, 4)
    bz, by, bx = np.meshgrid(*[np.arange(nb[a]) for a in (2, 1, 0)], indexing="ij")
    keys = brick_key(bx.ravel() + b0[0], by.ravel() + b0[1], bz.ravel() + b0[2])
    keep = (cb[..., 3] != 0).reshape(len(keys), -1).any(1)
    return keys[keep].astype(np.uint64), tb[keep], cb[keep]


def mesh_global(T, C, origin, cell, V, weight_cull=8):
    """mesh_oracle.mesh over the dense box of S (no border inside it), positions moved to the global lattice centred by V: (vertices,
    triangles, owners [n, 4] global).  Positions to mesh_oracle's tolerance."""
    n = T.shape[0]
    cell = np.float32(cell)
    v, t, own = mo.mesh(T, C, n, cell * np.float32(n), (0, 0, 0), tuple(int(x) for x in origin), (0, n, 0, n, 0, n), weight_cull,
                        return_owners=True)
    shift = np.float32(cell * n / 2 - cell * V / 2)
    for f in ("x", "y", "z"):
        v[f] = v[f] + shift
    own = own.copy(); own[:, :3] += np.asarray(origin, np.int64)
    return v, t, own


def open_edges(tris, keys=None):
    """Undirected edges used by exactly one triangle (vertex ids mapped through keys when given)."""
    t = np.asarray(tris, np.int64)
    if keys is not None:
        t = np.asarray(keys, np.int64)[t]
    e = np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]])
    e = np.sort(e, 1)
    u, c = np.unique(e, axis=0, return_counts=True)
    return u[c == 1]
