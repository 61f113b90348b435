"""numpy restatement of the map volume's restore (mapvol_restore_kernel in kintinuous_b200/csrc/kt_mapvol.cu), test-only, on top of
tests/map_volume_oracle.py's Store.

Once a shift has cleared its storage planes, every voxel of them whose global voxel (logical voxel + the wrap after the shift) lies in a
stored brick with W != 0 takes the stored tsdf and colour; every other voxel stays cleared."""
from __future__ import annotations

import numpy as np

import map_volume_oracle as mv


def restore(store, g):
    """The stored values of global voxels g int [n, 3]: (tsdf int16 [n], colour uint8 [n, 4], mask bool [n]), mask where a brick of
    `store` (map_volume_oracle.Store) holds the voxel with W != 0 (elsewhere tsdf and colour are 0)."""
    g = np.asarray(g, np.int64)
    b = g >> 3
    keys = mv.brick_key(b[:, 0], b[:, 1], b[:, 2])
    tsdf = np.zeros(len(g), np.int16); color = np.zeros((len(g), 4), np.uint8)
    uk, inv = np.unique(keys, return_inverse=True)
    for j, k in enumerate(uk):
        if int(k) not in store.bricks:
            continue
        idx = np.nonzero(inv == j)[0]
        l = g[idx] & 7
        t, c = store.bricks[int(k)]
        tsdf[idx] = t[l[:, 2], l[:, 1], l[:, 0]]
        color[idx] = c[l[:, 2], l[:, 1], l[:, 0]]
    mask = color[:, 3] != 0
    tsdf[~mask] = 0; color[~mask] = 0
    return tsdf, color, mask


def clear_planes(axis, back, V, current, delta):
    """The storage planes a clear from wrap `current` to `delta` along axis zeroes (kt_tsdf.cu's clear_range): |n| + 1 planes from the
    storage base (back: from base - |n|), on x at most round_up16(|n|) (Q13)."""
    an = abs(delta - current)
    base = current % V
    p0 = (base - an) % V if back else base
    count = an + 1
    if axis == 0:
        count = min(count, an if an % 16 == 0 else an + 16 - an % 16)
    return (p0 + np.arange(min(count, V))) % V


def shift_axis(store, tsdf, color, V, axis, planes, wrap, n, with_restore):
    """One axis of a shift on a storage-order volume, in place: store the planes, clear them and, with_restore, refill them from the
    store at the wrap after the shift.  Returns that wrap."""
    g, t, c, idx = mv.cleared_voxels(tsdf, color, V, axis, planes, wrap)
    store.clear(g, t, c)
    tsdf[idx] = 0; color[idx] = 0
    after = list(wrap); after[axis] += n
    if with_restore:
        g2, _, _, idx = mv.cleared_voxels(tsdf, color, V, axis, planes, after)
        rt, rc, m = restore(store, g2)
        tsdf[tuple(a[m] for a in idx)] = rt[m]; color[tuple(a[m] for a in idx)] = rc[m]
    return after
