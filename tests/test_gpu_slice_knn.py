"""Every output point of kt_op_process_slice (kt_slice.cu: weight cull, leaf grid, exact k-NN normals) against the numpy restatement in
tests/slice_knn_reference.py, scene by scene (SCENES below), on every point rather than a sample:

  * positions and colours bit for bit; alpha 0, data[3] = 1, data_n[3] = 0 and the padding 0;
  * normals within ANGLE_TOL rad of the FP64 reference (float32 output rounding ~6e-8 plus FP64 order and libm noise) on the points
    whose eigen-gap (lambda1 - lambda0) / lambda2 is at least GAP_MIN; a normal that lies in the plane through the viewpoint may take
    either sign; curvature within CURV_ULPS float32 ulps there, within 1e-6 everywhere; NaN normal and curvature with fewer than 3 neighbours;
  * the sheets show that the bound can see ONE wrong neighbour: swapping the k-th for the (k+1)-th moves most checked normals past it;
  * every scene sends its points down the search path it was built for (stop at r = 3 .. 10, cover, overflow past 768 candidates, R_CAP
    exhausted, isolated), and wherever the stop rule stopped, no point outside its cube had a key within the rule's reach (its premise,
    checked directly; the report gives the nearest such point per scene, against the margin the grid's extent gives the rule);
  * the output does not depend on the input order, bit for bit."""
import os
import sys

import numpy as np
import pytest

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tests"))
import slice_knn_reference as R  # noqa: E402
from slice_cloud import make_cloud  # noqa: E402

pytestmark = pytest.mark.gpu
ANGLE_TOL = 1e-6
GAP_MIN = 1e-3
CURV_ULPS = 4
SENSITIVE_MIN = 0.9


# ---- scenes: each one is built to send points down one of the search's paths (tests/slice_knn_reference.py names them).  Coordinates
# are exact multiples of the leaf where the leaf assignment must not depend on rounding; everything is seeded.
TRACKER_LEAF = float(np.float32(6.0 / 512))


def _points(xyz, rng, point_dtype):
    out = np.zeros(len(xyz), point_dtype)
    xyz = np.asarray(xyz, np.float32)
    out["x"], out["y"], out["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    for ch in ("r", "g", "b"):
        out[ch] = rng.integers(0, 256, len(xyz))
    out["a"] = rng.integers(8, 40, len(xyz))                                           # all kept at cull 8
    return out[rng.permutation(len(out))]


def sheet_at(centre, leaf, n_side=100, point_dtype=None):
    """make_cloud's sheet sampled at the leaf, moved so that its bounding box is centred on `centre` (one value for all axes)."""
    b = make_cloud(n_side=n_side, cell=leaf, offset=(0.0, 0.0, 0.0), point_dtype=point_dtype)
    xyz = np.stack([b["x"], b["y"], b["z"]], -1).astype(np.float64)
    mid = 0.5 * (xyz.min(0) + xyz.max(0))
    return make_cloud(n_side=n_side, cell=leaf, offset=tuple(float(centre) - mid), point_dtype=point_dtype)


def hollow_shell(leaf, point_dtype, n_hollow=2, hole=4.5, seed=7):
    """One jittered point per leaf in a block of leaves, with n_hollow^3 balls of `hole` leaves emptied around query points at their
    centres.  A query's +-4 cube holds nothing nearer than 4.5 leaves, so it cannot stop there, and its +-5 cube holds ~950 leaves,
    more than the 768 candidates the search keeps: the search overflows into the whole-cloud path."""
    rng = np.random.default_rng(seed)
    span = 14 * n_hollow + 2
    ijk = np.stack(np.meshgrid(*[np.arange(span)] * 3, indexing="ij"), -1).reshape(-1, 3)
    pos = ijk + rng.uniform(0.15, 0.85, ijk.shape)
    keep = np.ones(len(ijk), bool)
    centres = []
    for c in np.stack(np.meshgrid(*[np.arange(n_hollow)] * 3, indexing="ij"), -1).reshape(-1, 3):
        cc = 8 + 14 * c
        centres.append(cc + 0.5)
        keep &= np.linalg.norm(pos - (cc + 0.5), axis=1) > hole
        keep &= ~(ijk == cc).all(1)
    xyz = np.concatenate([pos[keep], np.array(centres)]) * leaf + 40 * leaf
    return _points(xyz, rng, point_dtype)


def sparse_lines(leaf, point_dtype, seed=3):
    """Thin ribbons of points, far from each other.  Along the axes the points are 2-3 leaves apart, so a +-10 cube holds fewer than
    20 of them; along the diagonal they are ~1.5 leaves apart, so a +-10 cube holds 20 or more, but the 20th lies ~14 leaves away.
    Either way the search runs out of radius (R_CAP = 10 leaves) without an isolated point in sight."""
    rng = np.random.default_rng(seed)
    lines = []
    for j, (axis, step) in enumerate([((1, 0, 0), 2.5), ((0, 1, 0), 2.5), ((0, 0, 1), 2.5), ((1, 1, 1), 1.5), ((1, 1, 1), 1.6), ((-1, 1, 1), 1.5)]):
        d = np.asarray(axis, np.float64) / np.linalg.norm(axis)
        u = np.cross(d, [0.3, 0.5, 0.8]); u /= np.linalg.norm(u); w = np.cross(d, u)
        t = np.cumsum(rng.uniform(step - 0.5 if step > 2 else step - 0.2, step + 0.5 if step > 2 else step + 0.2, 60))
        p = t[:, None] * d + rng.uniform(-1.0, 1.0, (60, 1)) * u + rng.uniform(-0.2, 0.2, (60, 1)) * w
        lines.append(p + np.array([40.0 * j, 200.0 - 30.0 * j, 100.0 + 40.0 * j]))
    return _points(np.concatenate(lines) * leaf, rng, point_dtype)


def tie_lattice(point_dtype, leaf=0.25, seed=11):
    """Points on an integer lattice of spacing (1, 1, 2) leaves with a power-of-two leaf: every coordinate, difference and squared
    distance is exact in float, so most points have several neighbours at exactly the distance of the 20th and the slot decides."""
    rng = np.random.default_rng(seed)
    ijk = np.stack(np.meshgrid(np.arange(12), np.arange(12), np.arange(0, 16, 2), indexing="ij"), -1).reshape(-1, 3)
    return _points(ijk * leaf + np.array([1.0, 2.0, 3.0]), rng, point_dtype)


def tiny_cloud(kind, leaf, point_dtype, seed=13):
    """Small clouds: 'box' fills 4 x 4 x 4 leaves (the search cube covers the grid from every leaf), 'few' has 7 points within
    3 x 3 x 3 leaves, 'spread' 12 points scattered over ~1 m (fewer than k points, never all in one search cube), 'two' and 'one'
    too few for a normal."""
    rng = np.random.default_rng(seed)
    base = 40 * leaf
    if kind == "box":
        xyz = base + rng.uniform(0.02, 3.98, (400, 3)) * leaf
    elif kind == "few":
        xyz = base + rng.uniform(0.02, 2.98, (7, 3)) * leaf
    elif kind == "spread":
        xyz = base + np.stack([np.arange(12) * 7.3, (np.arange(12) * 5) % 11 * 6.1, (np.arange(12) * 7) % 5 * 11.2], -1) * leaf + rng.uniform(0, 1, (12, 3)) * leaf
    else:
        xyz = base + rng.uniform(0.0, 30.0, ({"two": 2, "one": 1}[kind], 3)) * leaf
    return _points(xyz, rng, point_dtype)


def margin_sliver(point_dtype, copies=4):
    """With a 0.01 m leaf (inverse exactly 100) past x / leaf = 2^16, x * inv_leaf rounds on a 2^-7 grid, so a leaf boundary takes points
    up to 2^-8 leaf below it.  Q sits at x / leaf = 65534.99 (leaf 65534), A 4.999 leaves further along x but rounded into leaf 65540,
    outside Q's +-5 cube.  With k = 3 and B just inside 5 leaves, a stop rule whose margin is 0.001 leaf stops at r = 5 with {Q, P1, B};
    the exact set is {Q, P1, A}, whose normal is 90 degrees away.  The copies are 0.5 m apart along y."""
    q = np.array([10737254 * 2.0 ** -14, 0.3055, 0.4025])
    one = np.array([q, q + [819 * 2.0 ** -14, 0, 0], q - [0, 0.049989, 0], q + [0, 0, 0.015], q + [-0.3, 0.3, 0]])
    return _points(np.concatenate([one + [0, 0.5 * c, 0] for c in range(copies)]), np.random.default_rng(17), point_dtype)


def _power_of_two_centre(p2, leaf):
    """The coordinate where x * inverse_leaf crosses 2^p2 (float32 inverse, as the leaf grid computes it)."""
    return float(np.float32(2.0 ** p2) / (np.float32(1.0) / np.float32(leaf)))


# name -> (build(point_dtype), weight cull, leaf, k_search, {search path: least number of well-conditioned points that take it},
# sheet: the swap of the k-th for the (k+1)-th neighbour must show in the normals).  "ties": least number of points whose k-th and
# (k+1)-th neighbours are at exactly the same distance.
SCENES = {
    "sheet": (lambda d: make_cloud(point_dtype=d), 8, TRACKER_LEAF, 20, {"isolated": 8}, True),
    "sheet, no cull, leaf x2": (lambda d: make_cloud(point_dtype=d), 0, 2 * TRACKER_LEAF, 20, {"isolated": 8}, True),
    **{f"sheet at {s:+d} m": (lambda d, s=s: make_cloud(n_side=100, offset=(s, s, s), point_dtype=d), 8, TRACKER_LEAF, 20, {"stop4": 500}, True)
       for s in (100, -100, 800, -800, 1600, -1600)},
    **{f"sheet across x/leaf = 2^{p}, leaf {leaf:.6g}": (lambda d, p=p, leaf=leaf: sheet_at(_power_of_two_centre(p, leaf), leaf, point_dtype=d), 8, leaf, 20,
                                                         {"stop4": 500}, True)
       for leaf in (TRACKER_LEAF, 0.01) for p in (14, 15, 16)},
    "margin sliver at x/leaf = 2^16, leaf 0.01": (lambda d: margin_sliver(d), 8, 0.01, 3, {"stop6": 4}, False),
    "hollow shell": (lambda d: hollow_shell(TRACKER_LEAF, d), 8, TRACKER_LEAF, 20, {"overflow": 8}, False),
    "sparse lines": (lambda d: sparse_lines(TRACKER_LEAF, d), 8, TRACKER_LEAF, 20, {"rcap": 50, "isolated": 50}, False),
    "exact ties": (lambda d: tie_lattice(d), 8, 0.25, 20, {"ties": 500, "stop3": 1000}, False),
    "tiny box": (lambda d: tiny_cloud("box", TRACKER_LEAF, d), 8, TRACKER_LEAF, 20, {"covers": 60}, False),
    "7 points": (lambda d: tiny_cloud("few", TRACKER_LEAF, d), 8, TRACKER_LEAF, 20, {"covers": 7}, False),
    "12 scattered points": (lambda d: tiny_cloud("spread", TRACKER_LEAF, d), 8, TRACKER_LEAF, 20, {"isolated": 12}, False),
    "2 points": (lambda d: tiny_cloud("two", TRACKER_LEAF, d), 8, TRACKER_LEAF, 20, {}, False),
    "1 point": (lambda d: tiny_cloud("one", TRACKER_LEAF, d), 8, TRACKER_LEAF, 20, {}, False),
    **{f"sheet, k = {k}": (lambda d: make_cloud(n_side=80, point_dtype=d), 8, TRACKER_LEAF, k, {"stop3" if k < 32 else "stop4": 1000} if k >= 3 else {}, k >= 3)
       for k in (1, 2, 3, 19, 32)},
}


def _run_op(kb, pts, weight_cull, leaf, k):
    import torch
    from kintinuous_b200.binding import POINT_NORMAL_DTYPE
    d = torch.from_numpy(pts.view(np.uint8).reshape(-1).copy()).cuda()
    out = torch.zeros(max(1, len(pts)) * 48, dtype=torch.uint8, device="cuda")
    n = kb.ops.process_slice(d, len(pts), weight_cull, leaf, out, len(pts), k_search=k)
    return out.cpu().numpy().view(POINT_NORMAL_DTYPE)[:n].copy()


def _report(capsys, line):
    """one line per scene on the terminal, whether or not pytest captures output"""
    with capsys.disabled():
        print("\n" + line, end="")


def _angles(a, b, signed=True):
    """angle between unit vectors row by row, well conditioned near 0"""
    dot = (a * b).sum(1)
    return np.arctan2(np.linalg.norm(np.cross(a, b), axis=1), dot if signed else np.abs(dot))


@pytest.mark.parametrize("scene", list(SCENES))
def test_every_point_matches_the_exact_reference(built, scene, capsys):
    import kintinuous_b200 as kb
    from oracle.refbind import POINT_DTYPE
    build, cull, leaf, k, expect, sheet = SCENES[scene]
    pts = build(POINT_DTYPE)
    ref = R.process_slice(pts, cull, leaf, k)
    got = _run_op(kb, pts, cull, leaf, k)
    n, kk = len(ref["xyz"]), ref["kk"]
    assert len(got) == n, (scene, len(got), n)
    # positions and colours: bit for bit
    gxyz = np.stack([got["x"], got["y"], got["z"]], -1)
    bad = (gxyz.view(np.uint32) != ref["xyz"].view(np.uint32)).any(1)
    assert not bad.any(), (scene, int(bad.sum()), gxyz[bad][:3], ref["xyz"][bad][:3])
    for c, ch in enumerate("rgb"):
        assert np.array_equal(got[ch], ref["rgb"][:, c]), (scene, ch)
    assert (got["a"] == 0).all() and (got["_p0"] == 1.0).all() and (got["_p1"] == 0.0).all() and (got["_p2"] == 0.0).all()
    gn = np.stack([got["nx"], got["ny"], got["nz"]], -1).astype(np.float64)
    gc = got["curvature"].astype(np.float64)
    paths = np.bincount(ref["path"], minlength=len(R.PATHS))
    missing, checked = R.unmet(ref, expect, GAP_MIN)
    slack = ref["stop_slack"][np.isfinite(ref["stop_slack"])]
    line = (f"{scene}: {n} points, k {kk}, stop margin {ref['margin']:.4f} leaf, nearest point outside a stop cube "
            f"{f'r {float(slack.min()):+.5f}' if len(slack) else '-'} leaves")
    if kk < 3:
        assert np.isnan(gn).all() and np.isnan(gc).all(), scene
        _report(capsys, f"{line}: NaN normals as expected; paths {dict((p, int(c)) for p, c in zip(R.PATHS, paths) if c)}")
    else:
        assert np.isfinite(gn).all() and np.isfinite(gc).all(), scene
        x = ref["xyz"].astype(np.float64)
        # a normal (nearly) perpendicular to the ray from the viewpoint has no defined flip: compare it up to sign
        either = np.abs((x * ref["normal"]).sum(1)) <= 1e-9 * np.linalg.norm(x, axis=1)
        ang = np.where(either, _angles(gn, ref["normal"], signed=False), _angles(gn, ref["normal"]))
        rc = ref["curvature"]
        ulp = np.spacing(np.abs(rc).astype(np.float32)).astype(np.float64)
        dcu = np.abs(gc - rc) / ulp
        worst_ang = float(ang[checked].max()) if checked.any() else 0.0
        worst_cu = float(np.where(np.abs(gc - rc) <= 1e-12, 0.0, dcu)[checked].max()) if checked.any() else 0.0
        line += (f", {int(checked.sum())} checked, {int((~checked).sum())} excluded (eigen-gap < {GAP_MIN:g}), {int(either.sum())} with either sign; "
                 f"worst normal angle {worst_ang:.2e} rad, worst curvature {worst_cu:.2f} ulp ({np.abs(gc - rc).max():.1e} over all points)")
        if sheet:
            swapped = ref["slots"][:, :kk].copy()
            swapped[:, kk - 1] = ref["slots"][:, kk]
            alt, _, _ = R.normals(ref["xyz"], swapped)
            sens = float((_angles(alt, ref["normal"], signed=False)[checked] > ANGLE_TOL).mean())
            line += f"; one neighbour swapped moves {100 * sens:.1f} % of them past {ANGLE_TOL:g} rad"
        _report(capsys, f"{line}; paths of checked points {dict((p, int(c)) for p, c in zip(R.PATHS, np.bincount(ref['path'][checked], minlength=len(R.PATHS))) if c)}")
        far = checked & (ang > ANGLE_TOL)
        assert not far.any(), (scene, int(far.sum()), np.flatnonzero(far)[:5], ang[far][:5], [R.PATHS[p] for p in ref["path"][far][:5]])
        assert (np.abs(gc - rc) <= CURV_ULPS * ulp + 1e-12)[checked].all(), (scene, worst_cu)
        assert np.abs(gc - rc).max() <= 1e-6, scene
        if sheet:
            assert sens >= SENSITIVE_MIN, (scene, sens)
    # the stop rule's premise holds wherever it stopped, and the scene reaches what it was built for, on points whose output is checked
    assert not ref["stop_unsafe"].any() and not ref["stop_wrong"].any(), (scene, int(ref["stop_unsafe"].sum()), int(ref["stop_wrong"].sum()))
    assert not missing, (scene, missing)
    # input order does not matter, bit for bit
    again = _run_op(kb, pts[np.random.default_rng(1).permutation(len(pts))], cull, leaf, k)
    assert np.array_equal(got.view(np.uint8), again.view(np.uint8)), scene

