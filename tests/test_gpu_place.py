"""Loop detection on the GPU (kt_surf.cu, kt_place.cu, kt_detect_loops) against the restatement in oracle/place_oracle.py, and end to end on a
rendered trajectory that leaves its start and comes back.

Tolerances: SURF -- the same keypoints (the device and the oracle form the Hessian responses with the same float32 operations, so the
threshold and the 3 x 3 x 3 maxima are the same decisions), positions <= 1e-3 px, sizes <= 1e-4 relative, descriptors <= 1e-4 for >= 98 % of the keypoints
(continuous outputs in float32 vs FP64: a sample on a pixel boundary may round the other way); ratio matching -- exact indices and pass flags away from ties; PnP -- 1e-6 against the FP64 restatement; fitness -- 1e-5
relative against scipy's cKDTree."""
import sys

import numpy as np
import pytest

from conftest import ROOT

sys.path.insert(0, ROOT)
from oracle import place_oracle as PO  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def kb(built):
    import kintinuous_b200 as kb
    return kb


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _frame(k=5, cols=320, rows=240):
    from kintinuous_b200 import synth
    return synth.render(k, cols, rows, noise=True)


def test_surf_matches_oracle(kb):
    d, rgb = _frame()
    rows, cols = d.shape
    kp, desc = kb.ops.surf(_dev(rgb), rows, cols, max_features=300)
    okp, odesc = PO.surf(rgb, max_features=300)
    assert len(kp) == len(okp) and len(kp) > 20, (len(kp), len(okp))
    dpos = np.abs(kp[:, :2] - okp[:, :2]).max(1); dsz = np.abs(kp[:, 2] - okp[:, 2]) / okp[:, 2]
    w = int(np.argmax(dpos))
    assert dpos[w] <= 1e-3, (w, kp[w], okp[w])
    assert dsz.max() <= 1e-4, (int(np.argmax(dsz)), kp[np.argmax(dsz)], okp[np.argmax(dsz)])
    assert np.abs(kp[:, 4] - okp[:, 4]).max() <= 1e-4 * np.abs(okp[:, 4]).max()
    assert (kp[:, 5] == okp[:, 5]).all()
    dang = np.abs(np.angle(np.exp(1j * (kp[:, 3] - okp[:, 3]))))
    good = dang <= 1e-3
    assert good.mean() >= 0.98, good.mean()                 # an angle on a window edge may pick the neighbouring window
    # a descriptor sample whose rotated position lies on a pixel boundary may round to the neighbouring pixel in float32 vs FP64
    dd = np.abs(desc - odesc).max(1)
    assert (dd[good] <= 1e-4).mean() >= 0.98 and dd[good].max() <= 2e-3, (dd[good] > 1e-4).sum()
    kp2, desc2 = kb.ops.surf(_dev(rgb), rows, cols, max_features=300)
    assert np.array_equal(kp, kp2) and np.array_equal(desc, desc2)


def test_ratio_retrieval_counts_equal_brute_force(kb):
    # the retrieval as kt_detect_loops runs it: one segment per keyframe, only the first seg_counts[g] rows of a segment valid
    rng = np.random.default_rng(7)
    n_kf, per = 300, 40
    base = rng.standard_normal((per, 64)).astype(np.float32)
    db = rng.standard_normal((n_kf * per, 64)).astype(np.float32)
    db[123 * per:124 * per] = base + 0.05 * rng.standard_normal((per, 64)).astype(np.float32)      # one keyframe that matches
    db[200 * per:201 * per] = base + 0.05 * rng.standard_normal((per, 64)).astype(np.float32)      # ... and one that matches on 7 rows only
    db /= np.linalg.norm(db, axis=1, keepdims=True); q = base / np.linalg.norm(base, axis=1, keepdims=True)
    counts = rng.integers(0, per + 1, n_kf).astype(np.int32); counts[123] = per; counts[200] = 7; counts[5] = 0
    best, d1, d2, ps, seg = kb.ops.match_ratio(_dev(db), _dev(q), stride=per, seg_counts=counts)
    ob, od1, od2, ops_ = PO.match_ratio(db, q)
    valid = (np.arange(n_kf * per) % per) < np.repeat(counts, per)
    assert (best[~valid] == -1).all() and not ps[~valid].any()
    clear = valid & (np.abs(od1 - 0.49 * od2) > 1e-5)
    assert (best[valid] == ob[valid]).mean() > 0.999
    assert np.array_equal(ps[clear], ops_[clear])
    assert np.abs(d1[valid] - od1[valid]).max() < 1e-4
    ocount = (ops_ & valid).reshape(n_kf, per).sum(1); unclear = (valid & ~clear).reshape(n_kf, per).sum(1)
    assert np.array_equal(seg, ps.reshape(n_kf, per).sum(1))                  # the segmented sum is the flags' sum
    assert (np.abs(seg - ocount) <= unclear).all()
    assert seg[123] == ocount[123] and seg[200] == ocount[200] <= 7 and seg[5] == 0 and np.argmax(seg) == 123
    b2 = kb.ops.match_ratio(_dev(db), _dev(q), stride=per, seg_counts=counts)
    assert all(np.array_equal(x, y) for x, y in zip((best, d1, d2, ps, seg), b2))


def _pnp_set(seed, n=150, outliers=0.4):
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(seed)
    intr = np.array([264.0, 264.0, 160.0, 133.5])
    R = Rotation.from_rotvec(rng.normal(0, 0.2, 3)).as_matrix(); t = rng.normal(0, 0.2, 3)
    uv = np.stack([rng.uniform(10, 310, n), rng.uniform(10, 230, n)], 1); z = rng.uniform(1.0, 4.0, n)
    p_old = np.stack([(uv[:, 0] - intr[2]) * z / intr[0], (uv[:, 1] - intr[3]) * z / intr[1], z], 1)
    p_new = (p_old - t) @ R                          # R p_new + t = p_old
    uv_n = uv + rng.normal(0, 0.3, uv.shape)
    bad = rng.random(n) < outliers
    p_new[bad] += rng.normal(0, 0.5, (bad.sum(), 3))
    return p_new.astype(np.float32), p_old.astype(np.float32), uv_n.astype(np.float32), intr, R, t


def test_pnp_matches_oracle(kb):
    for seed in (1, 2, 3):
        pn, po, uv, intr, R, t = _pnp_set(seed)
        Rg, tg, inl, ni = kb.ops.pnp_ransac(pn, po, uv, intr)
        Ro, to, oinl = PO.pnp_ransac(pn, po, uv, intr)
        assert np.abs(Rg - Ro).max() < 1e-6 and np.abs(tg - to).max() < 1e-6, seed
        assert np.array_equal(inl, oinl) and ni == oinl.sum()
        assert np.abs(Rg - R).max() < 5e-3 and np.abs(tg - t).max() < 1e-2
        assert kb.ops.pnp_ransac(pn, po, uv, intr)[3] == ni and np.array_equal(kb.ops.pnp_ransac(pn, po, uv, intr)[0], Rg)


def test_cloud_fitness_matches_kdtree(kb):
    from kintinuous_b200 import synth
    from scipy.spatial.transform import Rotation
    cols, rows = 320, 240
    d0, _ = synth.render(0, cols, rows, noise=True); d1, _ = synth.render(6, cols, rows, noise=True)
    intr = synth.intrinsics(cols, rows)
    T = np.eye(4); T[:3, :3] = Rotation.from_rotvec([0.0, 0.02, 0.0]).as_matrix(); T[:3, 3] = [0.03, 0.0, 0.01]
    f, ns, nd = kb.ops.cloud_fitness(_dev(d0), _dev(d1), rows, cols, intr, 0.03, T)
    of, ons, ond = PO.fitness(d0, d1, intr, 0.03, T)
    assert (ns, nd) == (ons, ond)
    assert abs(f - of) <= 1e-5 * of + 1e-9, (f, of)
    assert kb.ops.cloud_fitness(_dev(d0), _dev(d1), rows, cols, intr, 0.03, T)[0] == f


# ---- end to end ----
COLS, ROWS = 320, 240


def _loop_pose(k, n_out=60):
    """Camera-to-world pose of frame k of a trajectory that turns and moves away for n_out frames, comes back over n_out and stays."""
    s = k if k <= n_out else max(0, 2 * n_out - k)
    a = np.deg2rad(0.6 * s)
    R = np.array([[np.cos(a), 0.0, np.sin(a)], [0.0, 1.0, 0.0], [-np.sin(a), 0.0, np.cos(a)]])
    return R, np.array([0.010 * s, 0.0, 0.004 * s])


_FRAMES = {}


def _run_sequence(kb, poses, detect, **params):
    from kintinuous_b200 import synth
    cfg = kb.Config.default(rows=ROWS, cols=COLS, vol=256)
    trk = kb.Tracker(cfg)
    if detect:
        trk.set_loop_detection(True, **params)
    out = []
    for k, (R, t) in enumerate(poses):
        key = (k, np.asarray(R).tobytes(), np.asarray(t).tobytes())
        if key not in _FRAMES:
            _FRAMES[key] = synth.render_at(R, t, COLS, ROWS, noise=True, noise_seed=k, texture=synth.cell_texture)
        d, c = _FRAMES[key]
        p = trk.process_frame(d, c, 33333 * (k + 1))
        out.append(np.concatenate([np.array(p.R), np.array(p.t), np.array(p.global_t)]).astype(np.float32))
    return trk, np.array(out)


def test_loop_detected_and_closed(kb):
    from scipy.spatial.transform import Rotation
    poses = [_loop_pose(k) for k in range(130)]
    # no throttle: the way back retraces the way out, so loops against the middle of the trajectory come first
    trk, _ = _run_sequence(kb, poses, True, exclude_recent=3, loop_throttle_s=0.0)
    n_kf, full = trk.num_keyframes()
    assert n_kf >= 6 and not full
    res = trk.detect_loops()
    assert len(res) == n_kf
    summary = [(r["keyframe"], r["stage_name"], r["candidate"], r["passes"], r["matches"], r["inlier_ratio"], r["fitness"]) for r in res]
    loops = [r for r in res if r["stage_name"] == "loop" and r["candidate"] <= 1]          # against an early keyframe
    assert loops, summary
    r = loops[0]
    assert r["closed"] == 1 and r["report"]["accepted"] == 1
    k1 = r["time"] // 33333 - 1; k2 = r["candidate_time"] // 33333 - 1
    R1, t1 = poses[k1]; R2, t2 = poses[k2]
    P1 = np.eye(4); P1[:3, :3] = R1; P1[:3, 3] = t1
    P2 = np.eye(4); P2[:3, :3] = R2; P2[:3, 3] = t2
    gt = np.linalg.inv(P1) @ P2
    C = r["constraint"]
    assert np.linalg.norm(C[:3, 3] - gt[:3, 3]) < 0.01
    assert np.degrees(np.linalg.norm(Rotation.from_matrix(C[:3, :3].T @ gt[:3, :3]).as_rotvec())) < 0.5
    assert r["fitness"] < 0.01 and len(r["inliers1"]) > 0
    t, dense, nf = trk.keyframe(r["keyframe"])
    assert t == r["time"] and nf > 40 and trk.dense_pose(dense)[2]
    trk.close()


def _sweep_pose(k):
    """A camera that turns on the spot, 1.5 degrees a frame: keyframes ~17 degrees apart, none revisited."""
    a = np.deg2rad(1.5 * k)
    return np.array([[np.cos(a), 0.0, np.sin(a)], [0.0, 1.0, 0.0], [-np.sin(a), 0.0, np.cos(a)]]), np.zeros(3)


def test_no_loop_without_revisit(kb):
    # exclude_recent = 4: every eligible keyframe looks more than 60 degrees away (the field of view is 62 degrees), so no loop may be
    # found; a candidate that retrieval lets through (random grey cells have look-alikes) must be rejected by the 3-D match count, the
    # PnP inlier ratio or the fitness check -- on this sequence one keyframe reaches the fitness check and fails it
    trk, _ = _run_sequence(kb, [_sweep_pose(k) for k in range(100)], True, exclude_recent=4)
    res = trk.detect_loops()
    stages = [(r["keyframe"], r["stage_name"], r["candidate"], r["passes"], r["matches"], r["inlier_ratio"], r["fitness"]) for r in res]
    assert len(res) >= 7
    assert all(r["stage_name"] in ("no_candidate", "matches", "inliers", "fitness") for r in res), stages
    assert all((r["candidate"] >= 0) == (r["stage_name"] != "no_candidate") for r in res), stages
    assert all(r["keyframe"] - r["candidate"] >= 4 for r in res if r["candidate"] >= 0), stages
    assert [r for r in res if r["stage_name"] == "fitness" and r["fitness"] >= 0.01], stages
    trk.close()


def _loops(res):
    return [(r["keyframe"], r["candidate"]) for r in res if r["stage_name"] == "loop"]


def test_rejected_loops_do_not_throttle_and_exclude_recent_holds(kb):
    poses = [_loop_pose(k) for k in range(130)]
    # the chi2 gate rejects every loop (isam_thresh ~ 0): the default 30 s throttle must not start, so later keyframes are still tried
    trk, _ = _run_sequence(kb, poses, True, exclude_recent=3, isam_thresh=1e-30)
    res = trk.detect_loops()
    loops = _loops(res)
    assert len(loops) >= 2, [(r["keyframe"], r["stage_name"]) for r in res]
    assert not [r for r in res if r["stage_name"] == "throttled"]
    assert all(r["closed"] == 0 and r["report"]["accepted"] == 0 for r in res if r["stage_name"] == "loop")
    assert trk.num_loops() == 0
    trk.close()
    # exclude_recent one above the smallest keyframe gap of those loops: that revisit is now inside the window, no loop has a smaller gap
    gap = min(q - c for q, c in loops)
    trk, _ = _run_sequence(kb, poses, True, exclude_recent=gap + 1, isam_thresh=1e-30)
    loops2 = _loops(trk.detect_loops())
    assert all(q - c >= gap + 1 for q, c in loops2), loops2
    assert not [l for l in loops2 if l in [(q, c) for q, c in loops if q - c == gap]]
    trk.close()


def test_accepted_loop_throttles(kb):
    # default 30 s throttle (frame timestamps): after the first ACCEPTED loop every later keyframe of this 4.3 s sequence is throttled
    trk, _ = _run_sequence(kb, [_loop_pose(k) for k in range(130)], True, exclude_recent=3)
    res = trk.detect_loops()
    i0 = next(i for i, r in enumerate(res) if r["stage_name"] == "loop")
    assert res[i0]["closed"] == 1 and i0 + 1 < len(res)
    assert all(r["stage_name"] == "throttled" for r in res[i0 + 1:]), [(r["keyframe"], r["stage_name"]) for r in res]
    trk.close()


def test_detection_does_not_change_tracking(kb):
    poses = [_loop_pose(k) for k in range(70)]
    a, pa = _run_sequence(kb, poses, False)
    b, pb = _run_sequence(kb, poses, True, exclude_recent=3)
    assert np.array_equal(pa, pb)
    ta, ca = a.export_volume(); tb, cb = b.export_volume()
    assert np.array_equal(ta, tb) and np.array_equal(ca, cb)
    assert a.num_slices() == b.num_slices()
    for i in range(a.num_slices()):
        assert np.array_equal(a.get_slice(i)[0], b.get_slice(i)[0])
    flags = []
    for i in range(a.num_dense_poses()):
        da, db = a.dense_pose(i), b.dense_pose(i)
        assert da[0] == db[0] and np.array_equal(da[1], db[1])
        flags.append(db[2])
    assert sum(flags) == b.num_keyframes()[0] and flags[0]
    b.detect_loops()
    a.close(); b.close()
