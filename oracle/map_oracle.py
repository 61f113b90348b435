"""TEST INFRASTRUCTURE ONLY (oracle/): never imported by the product path (kintinuous_b200/).

numpy restatement of the whole-map export (kt_map.cu, kt_get_map_cloud, kt_save_map_pcd):
  * voxel_grid -- pcl::VoxelGrid<PointT>::applyFilter of PCL 1.7.2 (filters/impl/voxel_grid.hpp) with downsample_all_data = true,
    min_points_per_voxel = 0, no filter field, is_dense = true, in float32: leaf i_k = int(floor(p_k * inv) - float(min_b_k)) with
    inv = 1.0f / leaf, the leaf index formed in 64 bits, a STABLE sort (points of a leaf in input order; PCL's std::sort leaves that
    order unspecified), every field summed in float32 from the first point on (NdCopyPointEigenFunctor: a -0.0 survives), divided by
    the float count, colour (int)r << 16 | (int)g << 8 | (int)b.  Works on POINT_DTYPE (x y z rgb) and POINT_NORMAL_DTYPE (x y z rgb
    normal_x normal_y normal_z curvature) records.
  * pcl_would_skip -- PCL's int64 overflow check (dx * dy * dz > INT_MAX: PCL returns the cloud unfiltered; kt_map.cu filters anyway).
  * the rigid correction of later slices (correction, rigid_move) in kt_tracker.cu's arithmetic.
  * the binary .pcd of PCL 1.7.2's savePCDFile(path, cloud, true) for PointXYZRGBNormal, restated from PCL's published
    PCDWriter::generateHeader / writeBinary.  UNPINNED against PCL itself (PCL is not installed here).
"""
import numpy as np

INT_MAX = 2 ** 31 - 1
PCD_FIELDS = ("x", "y", "z", "rgb", "normal_x", "normal_y", "normal_z", "curvature")


def _has_normals(pts):
    return "nx" in pts.dtype.names


def grid(pts, leaf):
    """(inv, min_b, div_b, pcl_would_skip) of VoxelGrid::applyFilter for a non-empty cloud (int64 numpy arrays for min_b / div_b)."""
    inv = np.float32(1.0) / np.float32(leaf)
    mn = np.array([pts[c].min() for c in "xyz"], np.float32)
    mx = np.array([pts[c].max() for c in "xyz"], np.float32)
    d = [int(np.float32(mx[a] - mn[a]) * inv) + 1 for a in range(3)]                 # static_cast<int64_t>((max - min) * inverse_leaf) + 1
    skip = d[0] * d[1] * d[2] > INT_MAX
    min_b = np.floor(mn * inv).astype(np.int64)
    div_b = np.floor(mx * inv).astype(np.int64) - min_b + 1
    return inv, min_b, div_b, bool(skip)


def leaf_ijk(pts, leaf):
    inv, min_b, _, _ = grid(pts, leaf)
    return [(np.floor(pts[c] * inv) - np.float32(min_b[a])).astype(np.int64) for a, c in enumerate("xyz")]


def leaf_keys(pts, leaf):
    """The 64-bit leaf index i0 + i1 div0 + i2 div0 div1 of every point."""
    _, _, div_b, _ = grid(pts, leaf)
    i0, i1, i2 = leaf_ijk(pts, leaf)
    return i0 + i1 * div_b[0] + i2 * (div_b[0] * div_b[1])


def pcl_index32(pts, leaf):
    """PCL's own int leaf index i0 * 1 + i1 * div0 + i2 * (div0 * div1), in int32 arithmetic."""
    _, _, div_b, _ = grid(pts, leaf)
    i0, i1, i2 = (a.astype(np.int32) for a in leaf_ijk(pts, leaf))
    with np.errstate(over="ignore"):
        d0 = np.int32(div_b[0]); d01 = np.int32(d0 * np.int32(div_b[1]))
        return i0 + i1 * d0 + i2 * d01


def _fold(v, starts, cnt):
    """Per leaf, the float32 left fold v[s] + v[s+1] + ... of its points in sorted order, starting at the first point."""
    acc = v[starts].copy()
    small = cnt <= 64
    kmax = int(cnt[small].max()) if small.any() else 0
    for k in range(1, kmax):
        sel = np.flatnonzero(small & (cnt > k))
        acc[sel] = acc[sel] + v[starts[sel] + k]
    for j in np.flatnonzero(~small):                                                     # np.add.accumulate is a sequential fold
        acc[j] = np.add.accumulate(v[starts[j]:starts[j] + cnt[j]])[-1]
    return acc


def voxel_grid(pts, leaf):
    """(centroids in ascending 64-bit leaf index, pcl_would_skip).  Same record type as pts."""
    if len(pts) == 0:
        return np.zeros(0, pts.dtype), False
    _, _, _, skip = grid(pts, leaf)
    keys = leaf_keys(pts, leaf)
    order = np.argsort(keys, kind="stable")
    ks = keys[order]
    head = np.ones(len(ks), bool)
    head[1:] = ks[1:] != ks[:-1]
    starts = np.flatnonzero(head)
    cnt = np.diff(np.append(starts, len(ks)))
    cntf = cnt.astype(np.float32)
    s = pts[order]
    names = ["x", "y", "z"] + (["nx", "ny", "nz", "curvature"] if _has_normals(pts) else [])
    out = np.zeros(len(starts), pts.dtype)
    for f in names:
        out[f] = _fold(np.ascontiguousarray(s[f], np.float32), starts, cnt) / cntf
    ch = {c: (_fold(s[c].astype(np.float32), starts, cnt) / cntf).astype(np.int32) for c in "rgb"}
    rgb = ((ch["r"] << 16) | (ch["g"] << 8) | ch["b"]).view(np.uint32)
    out["b"] = rgb & 0xff; out["g"] = (rgb >> 8) & 0xff; out["r"] = (rgb >> 16) & 0xff; out["a"] = rgb >> 24
    out["_p0"] = 1.0
    return out, skip


def correction(tracked, corrected):
    """C = P_corr P_tracked^-1 (4 x 4 float32 poses) as kt_tracker.cu forms it: FP64, rigid inverse, rounded to float32."""
    Pt = np.asarray(tracked, np.float32).reshape(4, 4).astype(np.float64).tolist()
    Pc = np.asarray(corrected, np.float32).reshape(4, 4).astype(np.float64).tolist()
    R = np.zeros((3, 3), np.float32); t = np.zeros(3, np.float32)
    for a in range(3):
        ta = Pc[a][3]
        for b in range(3):
            v = 0.0
            for k in range(3):
                v += Pc[a][k] * Pt[b][k]
            R[a, b] = v
            ta -= v * Pt[b][3]
        t[a] = ta
    return R, t


def rigid_move(pts, R, t):
    """x' = R x + t, n' = R n in float32, ((R0 x + R1 y) + R2 z) + t without contraction."""
    out = pts.copy()
    R = np.asarray(R, np.float32); t = np.asarray(t, np.float32)
    x, y, z = pts["x"], pts["y"], pts["z"]
    nx, ny, nz = pts["nx"], pts["ny"], pts["nz"]
    for a, c in enumerate("xyz"):
        out[c] = ((R[a, 0] * x + R[a, 1] * y) + R[a, 2] * z) + t[a]
        out["n" + c] = (R[a, 0] * nx + R[a, 1] * ny) + R[a, 2] * nz
    return out


def pcd_header(n):
    return ("# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS " + " ".join(PCD_FIELDS) + "\n"
            "SIZE 4 4 4 4 4 4 4 4\nTYPE F F F F F F F F\nCOUNT 1 1 1 1 1 1 1 1\n"
            f"WIDTH {n}\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS {n}\nDATA binary\n").encode()


PCD_BODY_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("b", "u1"), ("g", "u1"), ("r", "u1"), ("a", "u1"),
                           ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4"), ("curvature", "<f4")])
assert PCD_BODY_DTYPE.itemsize == 32


def pcd_bytes(pts):
    """The .pcd file of a POINT_NORMAL_DTYPE cloud."""
    body = np.zeros(len(pts), PCD_BODY_DTYPE)
    for f in PCD_BODY_DTYPE.names:
        body[f] = pts[f]
    return pcd_header(len(pts)) + body.tobytes()


def read_pcd(blob, point_dtype):
    """Parse a binary PointXYZRGBNormal .pcd (bytes) into point_dtype records (data[3] = 1 as PCL constructs the point)."""
    lines, off = {}, 0
    while True:
        end = blob.index(b"\n", off)
        line = blob[off:end].decode()
        off = end + 1
        if not line.startswith("#"):
            k, _, v = line.partition(" ")
            lines[k] = v
        if line.startswith("DATA"):
            break
    assert lines["DATA"] == "binary" and tuple(lines["FIELDS"].split()) == PCD_FIELDS, lines
    assert lines["SIZE"].split() == ["4"] * 8 and lines["TYPE"].split() == ["F"] * 8 and lines["COUNT"].split() == ["1"] * 8
    n = int(lines["POINTS"])
    assert int(lines["WIDTH"]) * int(lines["HEIGHT"]) == n and len(blob) - off == 32 * n
    body = np.frombuffer(blob, PCD_BODY_DTYPE, n, off)
    out = np.zeros(n, point_dtype)
    for f in PCD_BODY_DTYPE.names:
        out[f] = body[f]
    out["_p0"] = 1.0
    return out


def same_bits(a, b):
    """Records bit-identical, except that two NaNs in a float word match whatever their payloads (x86 keeps an operand's payload, the
    GPU returns the canonical NaN)."""
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    wa = np.ascontiguousarray(a).view(np.uint32).reshape(len(a), -1)
    wb = np.ascontiguousarray(b).view(np.uint32).reshape(len(b), -1)
    diff = wa != wb
    if not diff.any():
        return True
    fa, fb = wa.view(np.float32)[diff], wb.view(np.float32)[diff]
    return bool((np.isnan(fa) & np.isnan(fb)).all())
