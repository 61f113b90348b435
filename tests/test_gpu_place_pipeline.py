"""kt_detect_loops against oracle/place_oracle.py on the keyframes the tracker stored: for every keyframe, the oracle rebuilds its inputs
from the frames fed (matched by timestamp), pins SURF's keypoints, runs the retrieval (match_ratio + select_candidate) and verify, and the tracker's
candidate, pass count, match count and stage must be the oracle's; where a keyframe reaches PnP its inlier count and ratio, where it
reaches the dense check its fitness at the device's pose (1e-5 relative plus the derived float32 bound of the distances), its pose
against verify's (1e-5 m / 1e-5 rad, and then the fitness against verify's) and the back-projected inliers (bit for bit).  A decision
within float32 rounding -- a candidate or match set a ratio-test row within the derived bound can change, or the pose of a REJECTED
candidate whose ICP did not converge and whose FP64 association had pixels within rounding -- is reported and not compared; a loop's
pose is always compared.  The dense check's maps come from kt_op_frontend, the
front end the tracker runs on the stored keyframe depth."""
import sys

import numpy as np
import pytest

from conftest import ROOT

sys.path.insert(0, ROOT)
from oracle import place_oracle as PO  # noqa: E402

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
_FRAMES = {}


@pytest.fixture(scope="module")
def kb(built):
    import kintinuous_b200 as kb
    return kb


def _loop_pose(k, n_out):
    s = k if k <= n_out else max(0, 2 * n_out - k)
    a = np.deg2rad(0.6 * s)
    R = np.array([[np.cos(a), 0.0, np.sin(a)], [0.0, 1.0, 0.0], [-np.sin(a), 0.0, np.cos(a)]])
    return R, np.array([0.010 * s, 0.0, 0.004 * s])


def _frames(cols, rows, n_out, n):
    from kintinuous_b200 import synth
    key = (cols, rows, n_out, n)
    if key not in _FRAMES:
        _FRAMES[key] = [synth.render_at(*_loop_pose(k, n_out), cols, rows, noise=True, noise_seed=k, texture=synth.cell_texture) for k in range(n)]
    return _FRAMES[key]


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _maps(kb, depth, rgb, intr):
    import torch
    rows, cols = depth.shape
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    ds = [torch.zeros((rows >> l, cols >> l), dtype=torch.int16, device="cuda") for l in range(4)]
    vs = [torch.zeros((3 * (rows >> l), cols >> l), dtype=torch.float32, device="cuda") for l in range(4)]
    ns = [torch.zeros_like(v) for v in vs]
    kb.ops.frontend(dev(depth), dev(rgb), rows, cols, intr, 0, ds, vs, ns)
    return [(v.cpu().numpy().reshape(3, rows >> l, cols >> l), n.cpu().numpy().reshape(3, rows >> l, cols >> l)) for l, (v, n) in enumerate(zip(vs, ns))]


def _ratio_bound(d1, d2):
    g = 64 * U / (1 - 64 * U)
    r = float(np.float32(0.49))
    return ((2 * U + U * U) + g * (1 + 2 * U + U * U)) * (d1 + r * d2) + U * r * d2


def _fitness_bound(f, depth_old, depth_new, C):
    """How far a float32 fitness may lie from the FP64 one: every coordinate of a moved centroid and of its neighbour carries <= 8
    roundings of magnitude |p| + |t| (back-projection, centroid, transform, difference), so each distance d moves by at most delta and
    d^2 by 2 d delta + delta^2; the mean, by Cauchy-Schwarz, by 2 sqrt(f) delta + delta^2.  Plus 1e-5 relative for the sums."""
    zmax = max(int(depth_old.max()), int(depth_new.max())) / 1000.0
    delta = np.sqrt(3.0) * 8 * U * (2.0 * zmax + np.abs(np.asarray(C)[:3, 3]).sum())
    return 1e-5 * f + 2.0 * np.sqrt(f) * delta + delta * delta


def _run(kb, capsys, cols, rows, n_out, n, exclude_recent=3):
    from scipy.spatial.transform import Rotation
    frames = _frames(cols, rows, n_out, n)
    cfg = kb.Config.default(rows=rows, cols=cols, vol=256)
    trk = kb.Tracker(cfg)
    trk.set_loop_detection(True, exclude_recent=exclude_recent, loop_throttle_s=0.0, close=0)
    for k, (d, c) in enumerate(frames):
        trk.process_frame(d, c, 33333 * (k + 1))
    res = trk.detect_loops()
    n_kf, _ = trk.num_keyframes()
    assert len(res) == n_kf >= 4
    intr = np.array([cfg.fx, cfg.fy, cfg.cx, cfg.cy], np.float32)
    voxel = float(np.float32(cfg.volume_size) / np.float32(cfg.vol))
    kf, n_surf_pinned = [], 0
    for i in range(n_kf):
        t, _, nf = trk.keyframe(i)
        d, c = frames[t // 33333 - 1]
        # the keyframe's SURF: the oracle's keypoints must be the device's (count, order, positions); retrieval and verification then run
        # on the device's keypoints and descriptors, so that they are compared on the same inputs (the descriptors' own float32
        # tolerance is test_gpu_place_edges.py's)
        kp, desc = kb.ops.surf(_dev(c), rows, cols, max_features=1000)
        okp, _ = PO.surf(c, 1000)
        assert len(kp) == len(okp) == nf, (i, len(kp), len(okp), nf)
        assert np.abs(kp[:, :2] - okp[:, :2]).max() <= 1e-3 and np.array_equal(kp[:, 5], okp[:, 5]), i
        n_surf_pinned += len(kp)
        kf.append(dict(depth=d, rgb=c, kp=kp, desc=desc))
    lines, compared = [], dict(candidate=0, inliers=0, dense=0, pose=0, skipped=0)
    for r in res:
        q = r["keyframe"]
        nseg = q - exclude_recent + 1
        passes = np.zeros(q + 1, np.int64); amb = np.zeros(q + 1, np.int64)
        for g in range(max(nseg, 0)):
            _, d1, d2, ps = PO.match_ratio(kf[g]["desc"], kf[q]["desc"], float(np.float32(0.49)))
            passes[g] = ps.sum(); amb[g] = (np.abs(d1 - float(np.float32(0.49)) * d2) <= _ratio_bound(d1, d2)).sum()
        cand = PO.select_candidate(passes, q, exclude_recent, 40) if nseg > 0 else -1
        # the candidate is decided within rounding when a count within its ambiguous rows of the winner's, or of 40, could change it
        near = nseg > 0 and (any(abs(int(passes[g]) - int(passes[max(cand, 0)])) <= amb[g] + amb[max(cand, 0)] for g in range(nseg) if g != cand)
                             or abs(int(passes[:nseg].max()) - 40) <= amb[:nseg].max())
        line = f"kf {q}: device {r['stage_name']} cand {r['candidate']} passes {r['passes']} matches {r['matches']} inliers {r['inliers']} fitness {r['fitness']:.3g}"
        if near and r["candidate"] != cand:
            compared["skipped"] += 1
            lines.append(line + f" | oracle cand {cand} within rounding: skipped"); continue
        assert r["candidate"] == cand, (q, r["candidate"], cand, passes)
        if cand < 0:
            assert r["stage_name"] == "no_candidate", (q, r["stage_name"])
            lines.append(line); continue
        compared["candidate"] += 1
        assert r["passes"] == passes[cand] or abs(r["passes"] - passes[cand]) <= amb[cand], (q, r["passes"], passes[cand])
        o, nw = kf[cand], kf[q]
        v = PO.verify(o["depth"], o["kp"], o["desc"], nw["depth"], nw["kp"], nw["desc"], intr, _maps(kb, o["depth"], o["rgb"], intr),
                      _maps(kb, nw["depth"], nw["rgb"], intr), voxel, iterations=(10, 5, 4, 0))
        # rows of the pair's ratio test within float32 rounding of the 0.49 threshold or of their second neighbour may change the matches
        _, d1, d2, _ = PO.match_ratio(o["desc"], nw["desc"], float(np.float32(0.49)))
        B = _ratio_bound(d1, d2)
        amb_rows = int(((np.abs(d1 - float(np.float32(0.49)) * d2) <= B) | (d2 - d1 <= 2 * B)).sum())
        if r["matches"] != v["matches"] and amb_rows:
            compared["skipped"] += 1
            lines.append(line + f" | oracle matches {v['matches']}, {amb_rows} ratio rows within rounding: skipped"); continue
        assert r["matches"] == v["matches"], (q, r["matches"], v["matches"])
        assert r["stage_name"] == v["stage"] or (v["stage"] == "fitness" and r["stage_name"] == "loop" and abs(v["margin_fitness"]) < 1e-5 * v["fitness"]), (q, r["stage_name"], v["stage"])
        line += f" | oracle {v['stage']} matches {v['matches']}"
        if "inliers" in v:
            compared["inliers"] += 1
            assert r["inliers"] == v["n_inliers"] and r["inlier_ratio"] == np.float32(v["inlier_ratio"]), (q, r["inliers"], v["n_inliers"])
            line += f" inliers {v['n_inliers']}"
        if "C" in v:
            # the fitness stage on the device's own pose: the voxel grids and nearest neighbours of kt_slice.cu against the oracle's
            compared["dense"] += 1
            C_ = r["constraint"]
            f_at, _, _ = PO.fitness(o["depth"], nw["depth"], intr, float(np.float32(2.5) * np.float32(voxel)), C_.astype(np.float32))
            ftol = _fitness_bound(f_at, o["depth"], nw["depth"], C_)
            assert abs(r["fitness"] - f_at) <= ftol, (q, r["fitness"], f_at, ftol)
            # the pose: the dense ICP in float32 against verify's FP64 one
            dt = np.abs(C_[:3, 3] - v["C"][:3, 3]).max()
            dr = np.linalg.norm(Rotation.from_matrix(C_[:3, :3].T @ v["C"][:3, :3]).as_rotvec())
            line += f" fitness {v['fitness']:.6g} (device {r['fitness']:.6g}, oracle at device pose {f_at:.6g}), constraint err {dt:.2e} m {dr:.2e} rad, icp px within rounding {v['icp_ambiguous']}"
            if r["stage_name"] != "loop" and v["icp_ambiguous"] and (dt > 1e-5 or dr > 1e-5):
                # a rejected candidate: the alignment did not converge, and float32 and FP64 association decisions took it elsewhere
                compared["skipped"] += 1
                lines.append(line + ": rejected pose skipped"); continue
            assert dt <= 1e-5 and dr <= 1e-5, (q, dt, dr, v["icp_ambiguous"])
            assert abs(r["fitness"] - v["fitness"]) <= ftol, (q, r["fitness"], v["fitness"], ftol)
            compared["pose"] += 1
        if r["stage_name"] == "loop":
            assert np.array_equal(r["inliers1"], v["inliers1"]) and np.array_equal(r["inliers2"], v["inliers2"]), q
        lines.append(line)
    with capsys.disabled():
        print(f"\n[pipeline {cols}x{rows}] keyframes {n_kf}, keypoints pinned {n_surf_pinned}, " + ", ".join(f"{k} {v}" for k, v in compared.items()))
        for line in lines:
            print("  " + line)
    trk.close()
    return res, compared


def test_pipeline_320x240_out_and_back(kb, capsys):
    res, compared = _run(kb, capsys, 320, 240, 60, 130)
    assert compared["pose"] >= 1 and any(r["stage_name"] == "loop" for r in res)


def test_pipeline_640x480_out_and_back(kb, capsys):
    res, compared = _run(kb, capsys, 640, 480, 30, 66)
    assert compared["candidate"] >= 1
