"""Digests that let tests/golden/ pin large reference outputs bit for bit without storing them."""
import hashlib

import numpy as np


def raw(a):
    """SHA-256 of the array's bytes: equal digests mean bit-identical arrays."""
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def values(a):
    """SHA-256 of the array's values as np.array_equal(..., equal_nan=True) sees them: every NaN is one NaN and -0.0 equals 0.0."""
    a = np.array(a, copy=True)
    if a.dtype.kind == "f":
        a = a + a.dtype.type(0)
        a[np.isnan(a)] = np.nan
    return raw(a)


def vmap(a, rows, cols):
    """Digest of a 3-plane vertex / normal map where only plane 0 marks an invalid pixel (NaN): the other planes of an invalid pixel
    keep whatever the buffer held and are not part of the result."""
    m = np.array(a, np.float32, copy=True).reshape(3, rows, cols)
    m[:, np.isnan(m[0])] = np.nan
    return values(m)


def canon(pts):
    """32-byte points as a sorted multiset (rows of four uint64)."""
    a = np.ascontiguousarray(pts).view(np.uint64).reshape(len(pts), 4)
    return a[np.lexsort(a.T[::-1])] if len(a) else a
