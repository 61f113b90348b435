"""The normal equations of the odometry kernels against the FP64 reference (oracle/odometry_oracle.py), one pyramid level at a time.

KT_ODOM_ITERATIONS=0,..,1,..,0 makes a tracker run ONE iteration of ONE level, from the previous pose: exactly the system the oracle
rebuilds from the tracker's own inputs -- the model maps (download_map 2 / 3) before the frame, the current maps (0 / 1) after it, and
the photometric pyramids rebuilt from the two input frames with the kt_op_* chain (bit-identical to the tracker's fused front end,
test_gpu_ops.py::test_fused_frontend_equals_the_operator_chain).  Every level of odometry 0 (icp_frame_kernel), 1 and 2
(rgbd_frame_kernel<false / true>), on the whole-frame path and on the per-iteration kernels (KT_FORCE_PER_ITERATION, read once per
process: a subprocess), must give
  * the correspondence count and sum of squared intensity differences exactly (trace columns 43 / 42),
  * every A and b entry of the trace within the oracle's per-entry bound,
  * the pose after the one iteration within the bound propagated from the entries.
The scenes probe where the grid-wide fixed-point exchange of the sums could go wrong: magnitudes (a repeated frame, where the robust
scale sigma is 1 and the photometric sums reach ~1e13; a high-contrast checker close to the camera), correspondences confined to a few
CTAs, none at all, an int32-wrapping sum of squared differences, and the image widths on either side of the whole-frame kernel's
shared-memory stage."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import odometry_oracle as oo

pytestmark = pytest.mark.gpu

VOL = 128
LEVELS = 4


def _rgbd_max_k():
    """Chunks of 512 pixels per CTA that rgbd_frame_kernel stages, read from its source so that the stage-edge widths follow it."""
    import re
    from conftest import ROOT
    src = open(os.path.join(ROOT, "kintinuous_b200", "csrc", "kt_rgb.cu")).read()
    return int(re.search(r"\bRGBD_MAX_K\s*=\s*(\d+)", src).group(1))

_SCRIPT = r"""
import sys
import numpy as np
import kintinuous_b200 as kb
import os
src, dst, modes, levels = sys.argv[1], sys.argv[2], [int(m) for m in sys.argv[3].split(",")], [int(l) for l in sys.argv[4].split(",")]
f = np.load(src)
rows, cols = f["d0"].shape
out = {}
for mode in modes:
    for level in levels:
        it = [0] * 4; it[level] = 1
        os.environ["KT_ODOM_ITERATIONS"] = ",".join(str(v) for v in it)
        trk = kb.Tracker(kb.Config.default(rows=rows, cols=cols, vol=%d, odometry=mode))
        p0 = trk.process_frame(f["d0"], f["c0"], 0)
        key = f"{mode}_{level}"
        out[key + "_pose0"] = np.array(list(p0.R) + list(p0.t), np.float32)
        out[key + "_mv"] = trk.download_map(2, level); out[key + "_mn"] = trk.download_map(3, level)
        n0 = trk.launch_count()
        p1 = trk.process_frame(f["d1"], f["c1"], 1)
        out[key + "_launches"] = np.array(trk.launch_count() - n0)
        out[key + "_pose1"] = np.array(list(p1.R) + list(p1.t), np.float32)
        out[key + "_cv"] = trk.download_map(0, level); out[key + "_cn"] = trk.download_map(1, level)
        out[key + "_trace"] = trk.trace()
        trk.close()
np.savez(dst, **out)
""" % VOL


def _run(tmp_path, tag, frames, modes, levels, per_iteration):
    from conftest import ROOT
    src = str(tmp_path / f"{tag}_in.npz"); dst = str(tmp_path / f"{tag}_{int(per_iteration)}.npz")
    np.savez(src, d0=frames[0][0], c0=frames[0][1], d1=frames[1][0], c1=frames[1][1])
    env = dict(os.environ, PYTHONPATH=ROOT)
    env.pop("KT_FORCE_PER_ITERATION", None)
    if per_iteration:
        env["KT_FORCE_PER_ITERATION"] = "1"
    r = subprocess.run([sys.executable, "-c", _SCRIPT, src, dst, ",".join(map(str, modes)), ",".join(map(str, levels))],
                       env=env, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    return np.load(dst)


def _photometric_pyramids(frames, rows, cols):
    """Metric depth, intensity and gradient pyramids of both frames through the operator chain (cut-off 6 m, RGBDOdometry.cpp:147)."""
    import torch
    import kintinuous_b200 as kb
    ops = kb.ops
    out = []
    for d, c in frames:
        dd = torch.from_numpy(np.ascontiguousarray(d).view(np.int16)).cuda(); cc = torch.from_numpy(np.ascontiguousarray(c)).cuda()
        dm = [torch.zeros((rows >> l, cols >> l), dtype=torch.float32, device="cuda") for l in range(LEVELS)]
        im = [torch.zeros((rows >> l, cols >> l), dtype=torch.uint8, device="cuda") for l in range(LEVELS)]
        gx = [torch.zeros((rows >> l, cols >> l), dtype=torch.int16, device="cuda") for l in range(LEVELS)]
        gy = [torch.zeros((rows >> l, cols >> l), dtype=torch.int16, device="cuda") for l in range(LEVELS)]
        ops.short_depth_to_metres(dd, dm[0], rows, cols, 6000); ops.bgr_to_intensity(cc, im[0], rows, cols)
        for l in range(1, LEVELS):
            ops.pyrdown_gauss_f(dm[l - 1], dm[l], rows >> (l - 1), cols >> (l - 1))
            ops.pyrdown_uchar_gauss(im[l - 1], im[l], rows >> (l - 1), cols >> (l - 1))
        for l in range(LEVELS):
            ops.derivative_images(im[l], gx[l], gy[l], rows >> l, cols >> l)
        torch.cuda.synchronize()
        out.append(dict(depth=[t.cpu().numpy() for t in dm], image=[t.cpu().numpy() for t in im],
                        gx=[t.cpu().numpy() for t in gx], gy=[t.cpu().numpy() for t in gy]))
    return out


# ---------------------------------------------------------------------------------------------------------------------------------
# scenes: two frames each, frame 1 tracked against frame 0

def _synth(k, cols=640, rows=480):
    from kintinuous_b200 import synth
    return synth.render(k, cols, rows)


def _checker(shift):
    """A fronto-parallel plane at 0.5 m carrying a 0/255 checker of 8-pixel cells (shifted by `shift` pixels: a small motion)."""
    rows, cols = 480, 640
    y, x = np.mgrid[0:rows, 0:cols]
    v = np.where(((x + shift) // 8 + y // 8) % 2 == 0, 255, 0).astype(np.uint8)
    v = np.maximum(v, 1)                                 # intensity 0 is "no image" to the correspondence test
    return np.full((rows, cols), 500, np.uint16), np.repeat(v[..., None], 3, axis=2).copy()


def _scene(name):
    if name == "room":
        return [_synth(4), _synth(5)]
    if name == "repeated":
        return [_synth(4), _synth(4)]
    if name == "checker":
        return [_checker(0), _checker(1)]
    if name == "window":
        out = []
        for k in (4, 5):
            d, c = _synth(k)
            w = np.zeros_like(d); w[216:264, 296:344] = d[216:264, 296:344]
            out.append((w, c))
        return out
    if name == "black":
        d1, _ = _synth(5)
        return [_synth(4), (d1, np.zeros((480, 640, 3), np.uint8))]
    if name == "brighter":
        y, x = np.mgrid[0:480, 0:640]
        v = np.where((x // 2 + y // 2) % 2 == 0, 105, 1).astype(np.uint8)       # 2-pixel cells: every pixel passes the gradient test
        c0 = np.repeat(v[..., None], 3, axis=2).copy()
        d = np.full((480, 640), 1000, np.uint16)
        return [(d, c0), (d, (c0 + 150).astype(np.uint8))]
    raise ValueError(name)


# ---------------------------------------------------------------------------------------------------------------------------------

def _check(run, pyr, mode, level, rows, cols, report, tag):
    """Compare one (mode, level) run against the oracle: returns the list of failures (empty when it agrees) and appends a line to
    report."""
    from kintinuous_b200 import synth
    key = f"{mode}_{level}"
    fails = []
    kl, kd = oo.level_intrinsics(*synth.intrinsics(cols, rows), level)
    p0 = run[key + "_pose0"].astype(np.float64); Rp, tp = p0[:9].reshape(3, 3), p0[9:]
    p1 = run[key + "_pose1"].astype(np.float64); R1, t1 = p1[:9].reshape(3, 3), p1[9:]
    tr = run[key + "_trace"]
    if tr.shape[0] != 1:
        return [f"{tag} mode {mode} level {level}: {tr.shape[0]} trace rows, expected 1"]
    tr = tr[0].astype(np.float64)
    icp = oo.icp_system(run[key + "_cv"], run[key + "_cn"], run[key + "_mv"], run[key + "_mn"], Rp, tp, kl) if mode != 1 else None
    rgb = None
    if mode != 0:
        last, nxt = pyr[0], pyr[1]
        krk, kt = oo.build_warp(np.eye(4), *kd)
        corr = oo.photometric_correspondences(nxt["image"][level], nxt["depth"][level], nxt["gx"][level], nxt["gy"][level],
                                              last["depth"][level], last["image"][level], level, krk, kt)
        count, sigma_sq, n_amb = oo.count_and_sigma(corr)
        got_count, got_sigma = int(tr[43]), tr[42]
        if n_amb == 0:
            if got_count != count or got_sigma != float(np.float32(sigma_sq)):
                fails.append(f"{tag} mode {mode} level {level}: count / sigma^2 {got_count} / {got_sigma:.0f}, oracle {count} / {sigma_sq}")
            sigma = oo.q3_sigma(count, sigma_sq)
        else:
            # a tie in a correspondence test moves the count, hence sigma = sqrt(count) and every weight: the kernel's count must lie in
            # the oracle's range, and the rows are then weighted with the sigma of the kernel's own (checked) count
            if not count <= got_count <= count + n_amb:
                fails.append(f"{tag} mode {mode} level {level}: count {got_count}, oracle {count} .. {count + n_amb} ({n_amb} ambiguous)")
            sigma = oo.q3_sigma(got_count, 0 if got_sigma == 0 else 1)
        rgb = oo.photometric_system(corr, sigma, last["depth"][level], kl, kd)
    sys_tr = icp if mode == 0 else rgb                 # what the trace holds: the ICP system, or the photometric part alone
    A_tr = tr[:36].reshape(6, 6); b_tr = tr[36:42]
    # the trace stores float copies of the totals: half an ulp more
    errA = np.abs(A_tr - sys_tr.A) - (sys_tr.dA + np.abs(sys_tr.A) * oo.U)
    errb = np.abs(b_tr - sys_tr.b) - (sys_tr.db + np.abs(sys_tr.b) * oo.U)
    amax = float(np.abs(sys_tr.A).max())
    worst = float(max((np.abs(A_tr - sys_tr.A) / np.maximum(sys_tr.dA, 1e-300)).max(), (np.abs(b_tr - sys_tr.b) / np.maximum(sys_tr.db, 1e-300)).max()))
    if (errA > 0).any() or (errb > 0).any():
        i = np.unravel_index(np.argmax(np.abs(A_tr - sys_tr.A) - sys_tr.dA), (6, 6))
        fails.append(f"{tag} mode {mode} level {level}: A / b outside the bound by up to {worst:.3g}x; A{tuple(int(v) for v in i)} = "
                     f"{A_tr[i]:.9g}, oracle {sys_tr.A[i]:.9g} +- {sys_tr.dA[i]:.3g}; max|A| = {amax:.4g} = {amax / 2 ** 31:.3g} x 2^31")
    if mode == 0:
        if abs(tr[43] - icp.count) > icp.extra["ambiguous"]:
            fails.append(f"{tag} mode 0 level {level}: inliers {tr[43]:.0f}, oracle {icp.count} (+-{icp.extra['ambiguous']})")
        if abs(tr[42] - icp.residual) > icp.dres + abs(icp.residual) * oo.U:
            fails.append(f"{tag} mode 0 level {level}: residual {tr[42]:.9g}, oracle {icp.residual:.9g} +- {icp.dres:.3g}")
    full = icp if mode == 0 else rgb if mode == 1 else oo.merge(rgb, icp)
    Rc, tc, tol_R, tol_t, x = oo.pose_after_one_iteration(full, Rp, tp, guard=None if mode == 0 else 0.3)
    dR = float(np.abs(R1 - Rc).max()); dt = float(np.abs(t1 - tc).max())
    if dR > tol_R or dt > tol_t:
        fails.append(f"{tag} mode {mode} level {level}: pose |dR| {dR:.3g} (tol {tol_R:.3g}), |dt| {dt:.3g} (tol {tol_t:.3g})")
    report.append(f"{tag} mode {mode} level {level}: max|A| {amax:.4g} ({amax / 2 ** 31:.3g} x 2^31), worst entry {worst:.3g} of its bound, "
                  f"|dR| {dR:.2g}/{tol_R:.2g} |dt| {dt:.2g}/{tol_t:.2g}" + (f", count {rgb.count}" if rgb is not None else f", inliers {icp.count}"))
    return fails


@pytest.mark.parametrize("scene", ["room", "repeated", "checker", "window", "black", "brighter"])
def test_odometry_sums_match_the_fp64_oracle(built, tmp_path, scene):
    """(room) the synthetic room, frames 4 -> 5: the baseline at every level; (repeated) the same frame twice: every diff is 0, so
    sigma = 1 (Q3) and the photometric sums of levels 0-2 exceed 2^31; (checker) a 0/255 checker plane at 0.5 m moved by one pixel:
    the largest photometric magnitudes of the normal sigma regime; (window) depth only in a 48 x 48 window: all correspondences in one
    to three CTAs, the others add exact zeros; (black) the next image all zero: no photometric correspondence, so the photometric
    system is exactly zero; (brighter) a fine checker 150 levels brighter in the next frame: sum of diff^2 > 2^31, wrapped to int32
    as the reference does."""
    frames = _scene(scene)
    rows, cols = frames[0][0].shape
    pyr = _photometric_pyramids(frames, rows, cols)
    modes = [0, 1, 2]
    levels = list(range(LEVELS))
    fails, report = [], []
    for per_iteration in (False, True):
        run = _run(tmp_path, scene, frames, modes, levels, per_iteration)
        tag = f"{scene}/{'per-iteration' if per_iteration else 'whole-frame'}"
        for mode in modes:
            for level in levels:
                fails += _check(run, pyr, mode, level, rows, cols, report, tag)
                if scene == "black" and mode != 0:
                    tr = run[f"{mode}_{level}_trace"][0]
                    if tr.any():
                        fails.append(f"{tag} mode {mode} level {level}: photometric trace not exactly zero: {tr[np.nonzero(tr)][:6]}")
                    p0, p1 = run[f"{mode}_{level}_pose0"], run[f"{mode}_{level}_pose1"]
                    if mode == 1 and not np.array_equal(p0, p1):
                        fails.append(f"{tag} mode 1 level {level}: pose moved without correspondences: {p1 - p0}")
                if scene == "brighter" and mode != 0:
                    _check_wrapped_sigma(pyr, run[f"{mode}_{level}_trace"][0], level, rows, cols, fails, tag, mode)
    print("\n".join(report))
    assert not fails, "\n".join(fails)


def _check_wrapped_sigma(pyr, tr, level, rows, cols, fails, tag, mode):
    """The sum of squared differences wraps to int32 on both sides; kt_op_rgb_residual (residual_kernel) must agree with the trace."""
    import torch
    import kintinuous_b200 as kb
    from kintinuous_b200 import synth
    if level != 0:
        return
    _, kd = oo.level_intrinsics(*synth.intrinsics(cols, rows), level)
    krk, kt = oo.build_warp(np.eye(4), *kd)
    last, nxt = pyr[0], pyr[1]
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    cor = torch.zeros((rows * cols * 16,), dtype=torch.uint8, device="cuda")
    sigma, count = kb.ops.rgb_residual(float(np.float32(oo.MIN_GRADIENT[level] ** 2 / oo.SOBEL_SCALE ** 2)), dev(nxt["gx"][0]), dev(nxt["gy"][0]),
                                       dev(last["depth"][0]), dev(nxt["depth"][0]), dev(last["image"][0]), dev(nxt["image"][0]), cor, rows, cols,
                                       0.07, kt, krk)
    corr = oo.photometric_correspondences(nxt["image"][0], nxt["depth"][0], nxt["gx"][0], nxt["gy"][0], last["depth"][0], last["image"][0], 0, krk, kt)
    c, s, _ = oo.count_and_sigma(corr)
    exact = int((corr["diff"][corr["valid"]].astype(np.int64) ** 2).sum())
    if exact < 2 ** 31:
        fails.append(f"{tag} mode {mode}: the scene does not wrap the sum of squared differences ({exact})")
    if (sigma, count) != (s, c) or float(np.float32(s)) != float(tr[42]):
        fails.append(f"{tag} mode {mode}: kt_op_rgb_residual {sigma} / {count}, trace {tr[42]:.0f} / {tr[43]:.0f}, oracle {s} / {c} (exact {exact})")


def test_rgbd_stage_capacity_edge(built, tmp_path):
    """rgbd_frame_kernel stages RGBD_MAX_K (kt_rgb.cu) chunks of 512 pixels per CTA on min(SMs, 255) CTAs.  At 480 rows, the widest multiple-of-32
    image whose level 0 fits exactly takes the whole-frame kernel (one odometry launch); 32 columns more fall back to the per-iteration
    kernels.  Both must give the oracle's level-0 system (704 x 480 and 736 x 480 on a 132-SM H100 SXM, where 704 x 480 = 5 x 132 x 512)."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    G = min(sms, 255)
    rows = 480
    w_fit = (_rgbd_max_k() * G * 512 // rows) // 32 * 32
    launches = {}
    for cols in (w_fit, w_fit + 32):
        frames = [_synth(4, cols, rows), _synth(5, cols, rows)]
        pyr = _photometric_pyramids(frames, rows, cols)
        run = _run(tmp_path, f"edge{cols}", frames, [1, 2], [0], False)
        fails, report = [], []
        for mode in (1, 2):
            fails += _check(run, pyr, mode, 0, rows, cols, report, f"{cols}x{rows}")
            launches[(cols, mode)] = int(run[f"{mode}_0_launches"])
        print("\n".join(report))
        assert not fails, "\n".join(fails)
    for mode in (1, 2):
        # per-iteration level 0: point cloud + residual (+ ICP) + step launches in place of the one cooperative launch
        assert launches[(w_fit + 32, mode)] >= launches[(w_fit, mode)] + 2, (mode, launches)
