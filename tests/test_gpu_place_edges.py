"""Loop detection's operators at the edges where kernels go wrong, against oracle/place_oracle.py and brute force in FP64.

SURF (kt_op_surf) at the tracker's sizes 640x480 and 320x240 on rendered, textured, noisy frames: keypoint count, order, octave / layer
(through the size) and laplacian exact, positions <= 1e-3 px, sizes <= 1e-4 relative.  The angle and descriptor are continuous outputs of
float32 decisions: they must agree (angle <= 1e-4 rad, descriptor <= 1e-4) wherever the oracle's margins say float32 cannot flip a
decision -- the best window clear of the runner-up by more than float32 window sums can move it, no sample of the best window within
1e-4 degrees of its edge, no sample position within 1e-5 px or its float32 rounding bound of a rint boundary, and the measured angle
difference smaller than the turn that moves a descriptor sample to another pixel.  The keypoints under a margin are counted and
reported.  keypoints_3d (kt_op_keypoints_3d) bit for bit, ratio matching against an FP64 brute-force search outside a derived float32
bound, PnP to 1e-6 on degenerate and small sets, fitness to 1e-5 relative on clouds that straddle leaf boundaries."""
import sys

import numpy as np
import pytest

from conftest import ROOT

sys.path.insert(0, ROOT)
from oracle import place_oracle as PO  # noqa: E402

pytestmark = pytest.mark.gpu
U = 2.0 ** -24


@pytest.fixture(scope="module")
def kb(built):
    import kintinuous_b200 as kb
    return kb


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


_FRAMES = {}


def _report(capsys, line):
    """one line per case on the terminal, whether or not pytest captures output"""
    with capsys.disabled():
        print("\n" + line, end="")


def _frame(cols, rows, k=3):
    from kintinuous_b200 import synth
    key = (cols, rows, k)
    if key not in _FRAMES:
        _FRAMES[key] = synth.render_at(*synth.pose(k), cols, rows, noise=True, noise_seed=k, texture=synth.cell_texture)
    return _FRAMES[key]


def _tie_frame():
    """640x480 whose right half repeats its left half 320 px (a multiple of every octave's step) on: keypoints of equal response."""
    _, rgb = _frame(640, 480)
    rgb = rgb.copy(); rgb[:, 320:] = rgb[:, :320]
    return rgb


def _compare_surf(kb, capsys, rgb, max_features, label):
    rows, cols = rgb.shape[:2]
    kp, desc = kb.ops.surf(_dev(rgb), rows, cols, max_features=max_features)
    okp, odesc, mg = PO.surf(rgb, max_features=max_features, margins=True)
    assert len(kp) == len(okp), (label, len(kp), len(okp))
    n = len(kp)
    if n == 0:
        _report(capsys, f"[surf {label}] keypoints 0")
        return kp, okp
    # order, octave / layer (the nominal size of the refined one), response and laplacian: the same decisions
    assert np.array_equal(kp[:, 5], okp[:, 5]), label
    assert np.array_equal(kp[:, 4], okp[:, 4].astype(np.float32)), label
    dpos = np.abs(kp[:, :2] - okp[:, :2]).max(1)
    assert dpos.max() <= 1e-3, (label, int(np.argmax(dpos)), kp[np.argmax(dpos)], okp[np.argmax(dpos)])
    dsz = np.abs(kp[:, 2] - okp[:, 2]) / okp[:, 2]
    assert dsz.max() <= 1e-4, (label, int(np.argmax(dsz)))
    dang = np.abs(np.angle(np.exp(1j * (kp[:, 3].astype(np.float64) - okp[:, 3]))))
    under_ori = (mg["ori"] <= np.maximum(1e-5, mg["ori_bound"])) | (mg["ori_edge"] <= 1e-4)
    assert (dang[~under_ori] <= 1e-4).all(), (label, np.flatnonzero(~under_ori & (dang > 1e-4)))
    # the angle differs by dang: a sample moves by at most arm * dang (sample_turn), plus its float32 rounding (sample_slack)
    under_s = (mg["sample"] <= 1e-5) | (mg["sample_slack"] <= 0) | (mg["sample_turn"] <= dang + 4 * U)
    dd = np.abs(desc - odesc).max(1)
    clear = ~under_ori & ~under_s
    assert (dd[clear] <= 1e-4).all(), (label, np.flatnonzero(clear & (dd > 1e-4)), dd[clear].max())
    off = int(((dd > 1e-4) | (dang > 1e-4)).sum())
    _report(capsys, f"[surf {label}] keypoints {n} (device {len(kp)}), under orientation margin {int(under_ori.sum())}, under sample margin "
          f"{int((under_s & ~under_ori).sum())}, of those off by > 1e-4: {off}; max angle diff where clear {dang[~under_ori].max():.2e} rad, "
          f"max descriptor diff where clear {dd[clear].max() if clear.any() else 0:.2e}")
    # margins that flag everything would make this test blind
    assert clear.mean() >= 0.75, (label, clear.mean())
    return kp, okp


@pytest.mark.parametrize("cols,rows,max_features", [(640, 480, 100), (640, 480, 300), (640, 480, 1000), (320, 240, 100), (320, 240, 300),
                                                     (320, 240, 1000)])
def test_surf_at_the_trackers_sizes(kb, capsys, cols, rows, max_features):
    _, rgb = _frame(cols, rows)
    kp, _ = _compare_surf(kb, capsys, rgb, max_features, f"{cols}x{rows} max {max_features}")
    assert len(kp) >= min(max_features, 100)
    if cols == 640 and max_features == 1000:
        # octave 3's filters (side up to 216 px) have keypoints here
        assert (kp[:, 2] > 100).any()


def test_surf_cut_between_equal_responses(kb, capsys):
    rgb = _tie_frame()
    cands, _ = PO.detect(rgb)
    resp = np.array([-c[0][0] for c in cands])
    ties = np.flatnonzero(resp[:-1] == resp[1:])
    assert len(ties), "no equal responses"
    cut = int(ties[len(ties) // 2]) + 1                     # keeps the first of an equal pair, drops the second
    kp, okp = _compare_surf(kb, capsys, rgb, cut, f"tie cut at {cut}")
    assert len(kp) == cut and kp[-1, 4] == np.float32(resp[cut])


def test_surf_uniform_small_and_rotated(kb, capsys):
    flat = np.full((480, 640, 3), 128, np.uint8)
    kp, _ = kb.ops.surf(_dev(flat), 480, 640, max_features=300)
    assert len(kp) == 0
    # smaller than octave 3's largest filter (216 px): those layers are empty on both sides
    _, rgb = _frame(320, 240)
    small = np.ascontiguousarray(rgb[40:200, 60:260])
    kp, okp = _compare_surf(kb, capsys, small, 1000, "200x160")
    assert len(kp) > 10 and (kp[:, 2] < 150).all()
    rot = np.ascontiguousarray(np.rot90(rgb))
    kr, _ = _compare_surf(kb, capsys, rot, 300, "rotated 240x320")
    assert len(kr) > 20


def test_keypoints_3d_bit_identical(kb):
    rows, cols = 240, 320
    rng = np.random.default_rng(9)
    depth = rng.integers(300, 9000, (rows, cols)).astype(np.uint16)
    depth[rng.random((rows, cols)) < 0.1] = 0
    depth[10, 10:20] = 10000; depth[11, 10:20] = 12000; depth[12, 10:20] = 9999
    intr = np.array([264.0, 264.5, 159.5, 119.25], np.float32)
    h = np.float32(0.5)
    pts = []
    for u, v in [(12, 10), (15, 11), (13, 12), (0, 0), (cols - 1, 0), (0, rows - 1), (cols - 1, rows - 1)] + \
            [tuple(p) for p in rng.integers(0, (cols, rows), (40, 2))]:
        for d in (-h, h, np.nextafter(-h, np.float32(0)), np.nextafter(h, np.float32(0)), np.float32(0), np.float32(0.25)):
            pts.append((np.float32(u) + d, np.float32(v))); pts.append((np.float32(u), np.float32(v) + d))
    pts += [(-0.5, 3.0), (-0.49, 3.0), (cols - 0.5, 3.0), (cols - 0.51, 3.0), (3.0, rows - 0.5)]
    pts += [tuple(p) for p in rng.uniform(-2, (cols + 1, rows + 1), (2000, 2))]
    kp = np.zeros((len(pts), 6), np.float32); kp[:, :2] = np.array(pts, np.float32); kp[:, 2:] = 7.0
    got = kb.ops.keypoints_3d(_dev(kp), _dev(depth), rows, cols, intr)
    exp = PO.keypoints_3d(kp, depth, intr)
    assert np.array_equal(np.isnan(got), np.isnan(exp))
    assert np.array_equal(got.view(np.uint32)[~np.isnan(exp)], exp.view(np.uint32)[~np.isnan(exp)])
    assert np.isnan(got[:, 2]).sum() > 100 and (~np.isnan(got[:, 2])).sum() > 1000


def _brute(db, q):
    """FP64 squared distances of every db row to every q row, summed term by term (exact duplicates give exactly 0)."""
    out = np.empty((len(db), len(q)))
    for i in range(0, len(db), 256):
        out[i:i + 256] = ((db[i:i + 256, None, :].astype(np.float64) - q[None].astype(np.float64)) ** 2).sum(-1)
    return out


def _ratio_bound(d1, d2):
    """Float32 error of the device's decision d1 < fl(0.49f d2): each of the 64 terms e^2 with e = fl(a - b) is off by
    <= (2u + u^2) e^2, the 64 FMAs add <= gamma_64 of the (positive) sum, and the product 0.49f d2 rounds once."""
    g = 64 * U / (1 - 64 * U)
    term = (2 * U + U * U) + g * (1 + 2 * U + U * U)
    r = float(np.float32(0.49))
    return term * (d1 + r * d2) + U * r * d2


def test_match_ratio_edges(kb, capsys):
    rng = np.random.default_rng(21)
    per = 64
    q = rng.standard_normal((per, 64)).astype(np.float32); q /= np.linalg.norm(q, axis=1, keepdims=True)
    q[7] = q[3]; q[40] = q[41]                                           # exact duplicate queries: d1 == d2 for their nearest rows
    db = np.concatenate([q + 0.02 * rng.standard_normal(q.shape).astype(np.float32), rng.standard_normal((3 * per, 64)).astype(np.float32)])
    db /= np.linalg.norm(db, axis=1, keepdims=True)
    db[5] = q[3]                                                         # a row equal to a duplicated query: d1 = d2 = 0, no pass
    counts = np.array([per, 0, per, 17], np.int32)                       # seg_count == stride, 0 and partial
    r32 = float(np.float32(0.49))
    best, d1, d2, ps, seg = kb.ops.match_ratio(_dev(db), _dev(q), stride=per, seg_counts=counts)
    D = _brute(db, q)
    o = np.argsort(D, axis=1, kind="stable")
    od1 = D[np.arange(len(db)), o[:, 0]]; od2 = D[np.arange(len(db)), o[:, 1]]
    valid = (np.arange(len(db)) % per) < np.repeat(counts, per)
    assert (best[~valid] == -1).all() and not ps[~valid].any()
    B = _ratio_bound(od1, od2)
    clear = valid & (np.abs(od1 - r32 * od2) > B)
    assert np.array_equal(ps[clear], (od1 < r32 * od2)[clear])
    sure = valid & (od2 - od1 > 2 * B)
    assert np.array_equal(best[sure], o[sure, 0])
    assert (np.abs(d1[valid] - od1[valid]) <= 2 * B[valid] + 1e-30).all()
    assert d1[5] == 0.0 and d2[5] == 0.0 and not ps[5] and best[5] == 3     # ties: the lower index
    assert np.array_equal(seg, [ps[g * per:(g + 1) * per].sum() for g in range(4)]) and seg[1] == 0
    _report(capsys, f"[match_ratio] rows {valid.sum()}, within the float32 bound {int((valid & ~clear).sum())}")
    # a query set of one descriptor never passes
    best1, d11, d21, ps1, _ = kb.ops.match_ratio(_dev(db), _dev(q[:1]), stride=per, seg_counts=counts)
    assert not ps1.any() and (best1[valid] == 0).all()


def _pnp_set(seed, n, outliers=0.0, collinear=False):
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(seed)
    intr = np.array([264.0, 264.0, 160.0, 133.5])
    R = Rotation.from_rotvec(rng.normal(0, 0.2, 3)).as_matrix(); t = rng.normal(0, 0.2, 3)
    if collinear:
        s = rng.uniform(-1, 1, n)
        p_old = np.array([0.1, -0.05, 2.0]) + s[:, None] * np.array([0.3, 0.1, 0.2])
        uv = np.stack([intr[0] * p_old[:, 0] / p_old[:, 2] + intr[2], intr[1] * p_old[:, 1] / p_old[:, 2] + intr[3]], 1)
    else:
        uv = np.stack([rng.uniform(10, 310, n), rng.uniform(10, 230, n)], 1); z = rng.uniform(1.0, 4.0, n)
        p_old = np.stack([(uv[:, 0] - intr[2]) * z / intr[0], (uv[:, 1] - intr[3]) * z / intr[1], z], 1)
    p_new = (p_old - t) @ R
    uv_n = uv + rng.normal(0, 0.3, uv.shape)
    bad = np.zeros(n, bool); bad[:int(round(outliers * n))] = True
    p_new[bad] += rng.normal(0, 0.5, (bad.sum(), 3))
    return p_new.astype(np.float32), p_old.astype(np.float32), uv_n.astype(np.float32), intr


@pytest.mark.parametrize("case", ["n3", "collinear", "five_inliers", "all_inliers"])
def test_pnp_edges(kb, case):
    if case == "n3":
        pn, po, uv, intr = _pnp_set(31, 3)
    elif case == "collinear":
        pn, po, uv, intr = _pnp_set(32, 50, collinear=True)
    elif case == "five_inliers":
        pn, po, uv, intr = _pnp_set(33, 40, outliers=35 / 40)               # 5 good matches: fewer than 6, no refinement
    else:
        pn, po, uv, intr = _pnp_set(34, 120)
    Rg, tg, inl, ni = kb.ops.pnp_ransac(pn, po, uv, intr)
    Ro, to, oinl = PO.pnp_ransac(pn, po, uv, intr)
    assert np.abs(Rg - Ro).max() < 1e-6 and np.abs(tg - to).max() < 1e-6, (case, Rg, Ro, tg, to)
    assert np.array_equal(inl, oinl) and ni == oinl.sum(), case
    if case == "collinear":
        assert np.array_equal(Rg, np.eye(3)) and not tg.any() and ni == 0
    if case == "five_inliers":
        assert ni <= 5
    if case == "all_inliers":
        assert ni == len(pn)


@pytest.mark.parametrize("vol", [256, 512])
def test_fitness_edges(kb, vol):
    from kintinuous_b200 import synth
    from scipy.spatial.transform import Rotation
    cols, rows = 320, 240
    intr = synth.intrinsics(cols, rows)
    leaf = float(np.float32(2.5) * np.float32(6.0 / vol))
    d0, _ = _frame(cols, rows, 0); d1, _ = _frame(cols, rows, 9)
    # shift the second cloud's depths so that its centroid's z sits on a leaf boundary
    z = d1[d1 > 0].astype(np.float64).mean() / 1000.0
    k = np.round(z / leaf) * leaf
    d1 = np.where(d1 > 0, np.clip(d1.astype(np.int64) + int(round((k - z) * 1000)), 1, 65535), 0).astype(np.uint16)
    for rv, t in (([0.0, 0.0, 0.0], [0.0, 0.0, 0.0]), ([0.0, 0.25, 0.0], [0.4, 0.0, 0.1]), ([0.05, -0.3, 0.02], [-0.6, 0.1, 0.5])):
        T = np.eye(4); T[:3, :3] = Rotation.from_rotvec(rv).as_matrix(); T[:3, 3] = t
        T = T.astype(np.float32).astype(np.float64)
        f, ns, nd = kb.ops.cloud_fitness(_dev(d0), _dev(d1), rows, cols, intr, leaf, T)
        of, ons, ond = PO.fitness(d0, d1, intr, leaf, T)
        assert (ns, nd) == (ons, ond), (vol, rv)
        assert abs(f - of) <= 1e-5 * of + 1e-12, (vol, rv, f, of)
