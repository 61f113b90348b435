"""oracle/map_oracle.py (the checker of kt_map.cu and of the map export) pinned on the CPU: its float32 pcl::VoxelGrid against the slice
oracle's C++ restatement (oracle/kt_slice_oracle.cpp) and an independent float64 group-by, PCL's int64 overflow rule on both sides of
INT_MAX, the 64-bit key order against PCL's 32-bit index, and the .pcd layout."""
import os
import sys

import numpy as np
import pytest

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tests"))
from slice_cloud import make_cloud  # noqa: E402
from oracle import map_oracle as M  # noqa: E402
from oracle.refbind import POINT_DTYPE, POINT_NORMAL_DTYPE  # noqa: E402

LEAF = np.float32(6.0 / 512)


@pytest.fixture(scope="module")
def slice_oracle():
    from oracle import refbind
    import subprocess
    if not os.path.exists(os.path.join(ROOT, "oracle", "libkt_slice_oracle.so")):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "libkt_slice_oracle.so"])
    return refbind.SliceOracle()


@pytest.mark.parametrize("seed", [5, 6])
def test_voxel_grid_is_the_slice_oracles_bitwise(slice_oracle, seed):
    pts = make_cloud(seed=seed, point_dtype=POINT_DTYPE)
    want, _, _ = slice_oracle.voxel_grid(pts, float(LEAF))
    got, skip = M.voxel_grid(pts, LEAF)
    assert not skip and len(got) == len(want)
    for f in ("x", "y", "z"):
        assert got[f].tobytes() == want[f].tobytes(), f
    for f in ("r", "g", "b", "a", "_p0"):
        assert np.array_equal(got[f], want[f]), f


def test_voxel_grid_against_a_float64_group_by():
    rng = np.random.default_rng(3)
    pts = make_cloud(point_dtype=POINT_NORMAL_DTYPE)
    for c in ("nx", "ny", "nz", "curvature"):
        pts[c] = rng.uniform(-1, 1, len(pts)).astype(np.float32)
    got, _ = M.voxel_grid(pts, LEAF)
    ijk = np.stack(M.leaf_ijk(pts, LEAF), -1)
    uniq, inv, cnt = np.unique(ijk, axis=0, return_inverse=True, return_counts=True)
    inv = inv.reshape(-1)
    assert len(got) == len(uniq)
    # np.unique orders rows lexicographically by (i0, i1, i2); PCL's index orders them by (i2, i1, i0)
    order = np.lexsort((uniq[:, 0], uniq[:, 1], uniq[:, 2]))
    pos = np.empty(len(uniq), np.int64); pos[order] = np.arange(len(uniq))
    worst = 0.0
    for f in ("x", "y", "z", "nx", "ny", "nz", "curvature"):
        mean = np.bincount(inv, pts[f].astype(np.float64), len(uniq)) / cnt
        d = np.abs(got[f][pos].astype(np.float64) - mean).max()
        worst = max(worst, d)
    print(f"float32 fold vs float64 mean: {worst:.2e}")
    assert worst <= 1e-6
    for c in ("r", "g", "b"):
        mean = np.bincount(inv, pts[c].astype(np.float64), len(uniq)) / cnt
        assert (np.abs(got[c][pos].astype(np.float64) - mean) < 1.0).all()
    assert (got["a"] == 0).all() and (got["_p0"] == 1.0).all() and (got["_p1"] == 0).all()


def test_first_point_start_keeps_negative_zero_and_order_is_stable():
    pts = np.zeros(3, POINT_NORMAL_DTYPE)
    pts["x"] = [-0.0, 0.5, 0.25]; pts["y"] = [1.0, 1.0, 1.0]; pts["z"] = [2.0, 2.0, 2.0]
    pts["nx"] = [np.nan, 0.0, 0.0]
    got, _ = M.voxel_grid(pts, np.float32(0.1))
    assert len(got) == 3
    assert np.signbit(got["x"][0]) and got["x"][0] == 0.0                                # 0 + -0.0 would be +0.0
    assert np.isnan(got["nx"][0]) and not np.isnan(got["nx"][1:]).any()
    # one leaf of 1000 points: the left fold in input order, not numpy's pairwise sum
    rng = np.random.default_rng(1)
    one = np.zeros(1000, POINT_NORMAL_DTYPE)
    one["x"] = rng.uniform(3.0, 3.01, 1000).astype(np.float32); one["y"] = 1.0; one["z"] = 1.0
    got, _ = M.voxel_grid(one, np.float32(1.0))
    acc = np.float32(one["x"][0])
    for v in one["x"][1:]:
        acc = np.float32(acc + v)
    assert len(got) == 1 and got["x"][0] == np.float32(acc / np.float32(1000))


def test_pcl_would_skip_follows_the_int64_rule():
    def cloud(*corners):
        p = np.zeros(len(corners), POINT_DTYPE)
        p["x"], p["y"], p["z"] = np.asarray(corners, np.float32).T
        return p
    one = np.float32(1.0)
    # dx * dy * dz = 65536 * 32768 * 1 = 2^31 > INT_MAX; 65536 * 32767 = 2^31 - 65536 <= INT_MAX
    assert M.grid(cloud((0, 0, 0), (65535, 32767, 0)), one)[3]
    assert not M.grid(cloud((0, 0, 0), (65535, 32766, 0)), one)[3]
    # the check truncates (max - min) * inv, the grid floors each end: a span of 0.9 leaf is one cell to the check, two to the grid
    _, _, div_b, skip = M.grid(cloud((0.5, 0, 0), (1.4, 0, 0)), one)
    assert div_b[0] == 2 and not skip
    # the filter goes on past INT_MAX with 64-bit keys
    big = cloud((0, 0, 0), (65535, 32767, 0), (65535, 32767, 0), (1, 2, 0))
    got, skip = M.voxel_grid(big, one)
    assert skip and len(got) == 3 and got["x"][-1] == 65535.0


def test_key_order_is_pcls_below_int_max():
    pts = make_cloud(point_dtype=POINT_DTYPE)
    pts["x"] -= 3.0                                                                      # negative coordinates too
    _, _, div_b, skip = M.grid(pts, LEAF)
    assert not skip and int(np.prod(div_b)) <= M.INT_MAX
    k64 = M.leaf_keys(pts, LEAF); k32 = M.pcl_index32(pts, LEAF)
    assert np.array_equal(k64, k32.astype(np.int64))
    assert np.array_equal(np.argsort(k64, kind="stable"), np.argsort(k32, kind="stable"))


PCD_HEADER_7 = (b"# .PCD v0.7 - Point Cloud Data file format\n"
                b"VERSION 0.7\n"
                b"FIELDS x y z rgb normal_x normal_y normal_z curvature\n"
                b"SIZE 4 4 4 4 4 4 4 4\n"
                b"TYPE F F F F F F F F\n"
                b"COUNT 1 1 1 1 1 1 1 1\n"
                b"WIDTH 7\n"
                b"HEIGHT 1\n"
                b"VIEWPOINT 0 0 0 1 0 0 0\n"
                b"POINTS 7\n"
                b"DATA binary\n")


def test_pcd_layout_and_round_trip(tmp_path):
    rng = np.random.default_rng(2)
    pts = np.zeros(7, POINT_NORMAL_DTYPE)
    for f in ("x", "y", "z", "nx", "ny", "nz", "curvature"):
        pts[f] = rng.normal(size=7).astype(np.float32)
    for f in ("r", "g", "b", "a"):
        pts[f] = rng.integers(0, 256, 7)
    pts["_p0"] = 1.0
    blob = M.pcd_bytes(pts)
    assert blob[:len(PCD_HEADER_7)] == PCD_HEADER_7 and len(blob) == len(PCD_HEADER_7) + 7 * 32
    body = blob[len(PCD_HEADER_7):]
    assert body[:12] == pts[:1]["x"].tobytes() + pts[:1]["y"].tobytes() + pts[:1]["z"].tobytes()
    assert body[12:16] == bytes([pts["b"][0], pts["g"][0], pts["r"][0], pts["a"][0]])      # rgb: b, g, r, a
    path = tmp_path / "map.pcd"
    path.write_bytes(blob)
    back = M.read_pcd(path.read_bytes(), POINT_NORMAL_DTYPE)
    assert back.tobytes() == pts.tobytes()
    assert M.read_pcd(M.pcd_bytes(pts[:0]), POINT_NORMAL_DTYPE).size == 0
