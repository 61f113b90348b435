"""GPU parity tests, tracker level (kt_create / kt_process_frame / kt_finalise through the C ABI).
Bar (BASELINE.json north_star): pose <= 1e-4 m / 1e-4 rad against the reference's CUDA path on the same synthetic RGB-D input;
TSDF <= 1 LSB.  Per operator the TSDF is bit-exact (test_gpu_ops.py); over a sequence the pose differs by ~1e-6 (the ICP sums use a
different summation tree), which moves a few voxel projections across a pixel boundary, so the sequence-level TSDF bar is stated as
a fraction of voxels within 1 LSB."""
import os

import numpy as np
import pytest

from conftest import GOLDEN

pytestmark = pytest.mark.gpu


def rot_angle(Ra, Rb):
    d = Ra.astype(np.float64) @ Rb.astype(np.float64).T
    w = np.array([d[2, 1] - d[1, 2], d[0, 2] - d[2, 0], d[1, 0] - d[0, 1]]) * 0.5
    return float(np.linalg.norm(w))          # sin(angle), accurate near zero (arccos of the trace is not)


@pytest.fixture(scope="module")
def frames():
    from kintinuous_b200 import synth
    return [synth.render(k) for k in range(10)]


@pytest.mark.parametrize("name,kw,nframes", [("icp", dict(odometry=0), 10), ("icp_shift", dict(odometry=0, voxel_shift=2), 10), ("icp_rgbd", dict(odometry=2), 4)])
def test_tracker_vs_golden_reference_cuda(built, frames, name, kw, nframes):
    import kintinuous_b200 as kb
    g = np.load(os.path.join(GOLDEN, f"tracker_{name}_256.npz"))
    trk = kb.Tracker(kb.Config.default(vol=256, **kw))
    for k in range(nframes):
        p = trk.process_frame(frames[k][0], frames[k][1], k)
        R, t, gc, w = p.as_tuple()
        gp = g["poses"][k]
        assert np.abs(t - gp[9:12]).max() <= 1e-4, (name, k)
        assert rot_angle(R, gp[:9].reshape(3, 3)) <= 1e-4, (name, k)
        assert np.abs(gc - gp[12:15]).max() <= 1e-4
        assert (w == gp[15:18].astype(np.int32)).all()
        if k in (1, 2):
            tr = trk.trace(); gt = g[f"trace{k}"]
            assert len(tr) == len(gt)
            rel = np.abs(tr[:, :42] - gt[:, :42]).max(1) / np.abs(gt[:, :42]).max(1)
            assert rel.max() < 2e-3, (name, k, rel.max())
    if nframes == 10:
        ts, cs = trk.export_volume()
        touched = int((cs[..., 3] != 0).sum())
        assert abs(touched - int(g["touched"])) <= 2e-3 * int(g["touched"])
        hist = np.bincount((ts.reshape(-1)[cs[..., 3].reshape(-1) != 0].astype(np.int32) + 32768) >> 8, minlength=256)
        assert np.abs(hist - g["tsdf_hist"]).sum() <= 0.01 * touched
        trk.finalise()
        gs = g["slices"]
        assert trk.num_slices() == len(gs)
        for i in range(len(gs)):
            pts, dim, cam_t = trk.get_slice(i)
            assert dim == gs[i][0]
            info = trk.slice_info(i)                                   # the full CloudSlice record
            assert info.dimension == dim and info.count == len(pts) and info.odometry == (0 if kw.get("odometry", 0) == 0 else 2)
            assert np.allclose(np.array(info.camera_t), cam_t) and abs(np.linalg.det(np.array(info.camera_R).reshape(3, 3)) - 1) < 1e-3
            # the reference's count of a full-volume extraction can be a few points short (its publication race, DESIGN.md R1)
            assert abs(len(pts) - gs[i][1]) <= max(5, 0.01 * gs[i][1]), (i, len(pts), gs[i])
    trk.close()


def test_tracker_vs_reference_cuda_live(built, frames):
    """Frame by frame against the reference tracker's run on the same input (tests/golden/ref_tracker_live_256.npz: its poses, a seeded
    sample of 50 000 of its touched voxels, its model maps' invalid-pixel masks and a sample of their valid pixels)."""
    import kintinuous_b200 as kb
    g = np.load(os.path.join(GOLDEN, "ref_tracker_live_256.npz"))
    cfg = kb.Config.default(vol=256)
    mine = kb.Tracker(cfg)
    for k, (d, c) in enumerate(frames):
        p = mine.process_frame(d, c, k)
        Ra, ta, ga, wa = p.as_tuple(); Rb, tb, wb = g["poses"][k][:9].reshape(3, 3), g["poses"][k][9:12], g["wraps"][k]
        assert np.abs(ta - tb).max() <= 1e-4 and rot_angle(Ra, Rb) <= 1e-4 and (wa == wb).all()
    ta, ca = mine.export_volume()
    idx = g["vol_idx"]
    d = np.abs(ta.reshape(-1)[idx].astype(np.int32) - g["vol_tsdf"].astype(np.int32))
    assert (d <= 1).mean() >= 0.995, float((d <= 1).mean())      # poses differ by ~1e-6
    assert (ca[..., 3].reshape(-1)[idx] == g["vol_weight"]).mean() >= 0.999
    # model maps handed to the next frame (raycast + in-kernel pyramid vs raycast + 6 resize launches)
    for lvl in range(3):
        va = mine.download_map(2, lvl)
        na = np.isnan(va[0]).reshape(-1)
        nb = np.unpackbits(g[f"map_nan_{lvl}"], count=na.size).astype(bool)
        assert (na != nb).mean() < 2e-3
        px = g[f"map_px_{lvl}"]
        ok = ~na[px]
        assert np.quantile(np.abs(va.reshape(3, -1)[:, px[ok]] - g[f"map_v_{lvl}"][:, ok]).max(0), 0.999) < 1e-3
    mine.close()


@pytest.mark.parametrize("odometry", [0, 2])
def test_degenerate_frames_vs_reference_cuda_live(built, frames, odometry):
    """Edge cases the domain has, frame by frame against the reference's CUDA path: depth with holes and sensor noise, a completely
    empty depth frame (no ICP inliers: the 6x6 system is all zeros and the solve must return a zero increment like Eigen's LDLT),
    a half-empty frame, and a repeated frame (zero motion).  The reference's run: tests/golden/ref_degenerate_256.npz (its poses and,
    ICP-only, a seeded sample of 100 000 of its touched voxels)."""
    import kintinuous_b200 as kb
    from kintinuous_b200 import synth
    g = np.load(os.path.join(GOLDEN, "ref_degenerate_256.npz"))
    rng = np.random.default_rng(11)
    seq = []
    for k in range(8):
        d, c = synth.render(k, noise=True) if k in (1, 2) else frames[k]
        d = d.copy()
        if k == 3:
            d[:] = 0                                              # empty frame
        if k == 4:
            d[:, 320:] = 0                                        # half of the image without depth
        if k == 5:
            d[rng.random(d.shape) < 0.3] = 0                      # 30 % holes
        if k == 6:
            d, c = seq[-1]                                        # the same frame again
        seq.append((d, c))
    cfg = kb.Config.default(vol=256, odometry=odometry)
    mine = kb.Tracker(cfg)
    for k, (d, c) in enumerate(seq):
        p = mine.process_frame(d, c, k)
        Ra, ta, ga, wa = p.as_tuple()
        gp = g[f"poses_{odometry}"][k]; Rb, tb, wb = gp[:9].reshape(3, 3), gp[9:12], g[f"wraps_{odometry}"][k]
        assert np.isfinite(ta).all() and np.isfinite(Ra).all(), k
        tol = 1e-4 if (odometry == 0 or k < 3) else 2e-3          # photometric odometry is chaotic after a few frames (DESIGN.md section 5)
        assert np.abs(ta - tb).max() <= tol and rot_angle(Ra, Rb) <= tol and (wa == wb).all(), (k, np.abs(ta - tb).max())
    ta, ca = mine.export_volume()
    if odometry == 0:
        d = np.abs(ta.reshape(-1)[g["vol_idx"]].astype(np.int32) - g["vol_tsdf"].astype(np.int32))
        assert (d <= 1).mean() >= 0.99, float((d <= 1).mean())
        assert abs(int((ca[..., 3] != 0).sum()) - int(g["touched"])) <= 2e-3 * int(g["touched"])
    mine.close()


def test_run_to_run_determinism(built, frames):
    """Fixed-order reductions: two runs give bit-identical poses and volumes (the reference's own reductions are deterministic too)."""
    import kintinuous_b200 as kb
    outs = []
    for _ in range(2):
        trk = kb.Tracker(kb.Config.default(vol=256))
        poses = []
        for k in range(6):
            p = trk.process_frame(frames[k][0], frames[k][1], k)
            poses.append(np.concatenate([np.array(p.R), np.array(p.t)]))
        ts, cs = trk.export_volume()
        outs.append((np.array(poses), ts.copy(), cs.copy()))
        trk.close()
    assert (outs[0][0].view(np.uint32) == outs[1][0].view(np.uint32)).all()
    assert (outs[0][1] == outs[1][1]).all() and (outs[0][2] == outs[1][2]).all()


def test_device_and_host_entry_points_agree(built, frames):
    import torch
    import kintinuous_b200 as kb
    a = kb.Tracker(kb.Config.default(vol=256)); b = kb.Tracker(kb.Config.default(vol=256))
    for k in range(4):
        d, c = frames[k]
        pa = a.process_frame(d, c, k)
        pb = b.process_frame_device(torch.from_numpy(d.view(np.int16)).cuda(), torch.from_numpy(c).cuda(), k)
        assert list(pa.t) == list(pb.t) and list(pa.R) == list(pb.R)
    a.close(); b.close()


def test_full_size_properties_512(built, frames):
    """BASELINE size (640x480 into 512^3): size-independent properties instead of an oracle run --
    integrate is idempotent in its support (second integration of the same frame touches the same voxels and only raises weights),
    a cleared slab extracts no points, extraction count is invariant under the cyclic storage offset."""
    import torch
    import kintinuous_b200 as kb
    from kintinuous_b200 import synth
    V = 512
    rows, cols = 480, 640
    ops = kb.ops
    intr = np.array(synth.intrinsics(cols, rows), np.float32)
    d, c = frames[0]
    dd = torch.from_numpy(d.view(np.int16)).cuda(); cc = torch.from_numpy(c).cuda()
    fb = torch.zeros((rows, cols), dtype=torch.int16, device="cuda"); ops.bilateral(dd, fb, rows, cols)
    vm = torch.zeros((3 * rows, cols), dtype=torch.float32, device="cuda"); nm = torch.zeros_like(vm)
    ops.create_maps(intr, fb, vm, nm, rows, cols)
    trunc = 0.06
    vs = [6.0] * 3
    R = np.eye(3, dtype=np.float32); t = np.array([3, 3, 3], np.float32)
    results = []
    for wrap in ((0, 0, 0), (37, 501, 255)):
        ts = torch.zeros(V ** 3, dtype=torch.int16, device="cuda"); cs = torch.zeros(V ** 3 * 4, dtype=torch.uint8, device="cuda")
        ops.init_volume(ts, cs, V)
        ds = torch.zeros((rows, cols), dtype=torch.float32, device="cuda")
        ops.integrate(dd, rows, cols, intr, vs, R, t, trunc, ts, cs, V, wrap, cc, nm, 1, ds)
        w1 = cs.view(-1, 4)[:, 3].clone(); t1 = ts.clone()
        ops.integrate(dd, rows, cols, intr, vs, R, t, trunc, ts, cs, V, wrap, cc, nm, 1, ds)
        w2 = cs.view(-1, 4)[:, 3]
        assert bool(((w1 != 0) == (w2 != 0)).all()) and bool((w2[w1 != 0] == 2).all())
        assert int((ts.to(torch.int32) - t1.to(torch.int32)).abs().max().item()) <= 1          # mean of two equal samples
        cap = 3 * rows * cols
        out = torch.zeros(cap * 32, dtype=torch.uint8, device="cuda")
        n_full = ops.extract_slice(ts, vs, V, out, cap, wrap, cs, (0, V, 0, V, 0, V), 1, (0, 0, 0))
        results.append((int((w2 != 0).sum().item()), n_full))
        ops.clear_volume(2, 0, ts, cs, V, wrap[2], wrap[2] + 500)                                # logical z planes [0, 500]
        assert ops.extract_slice(ts, vs, V, out, cap, wrap, cs, (0, V, 0, V, 0, 499), 1, (0, 0, 0)) == 0
    assert results[0] == results[1]                                                              # cyclic offset changes storage, not content


@pytest.mark.parametrize("odometry", [0, 1, 2])
def test_prefetch_hint_does_not_change_results(built, frames, odometry):
    """kt_prefetch_frame moves the copy AND the pose-independent front end of the next frame (scaleDepth, bilateral, pyramid, maps, and
    for -r / -ri the photometric pyramids) onto a side stream, into a spare buffer set.  Results must be bit-identical with the hint,
    without it, with hints given only for some frames, and with a hint before the first frame (it copies the inputs only) -- including
    the stale y/z planes of invalid map pixels (Q7) that the colour integration can read, hence the depth holes."""
    import torch
    import kintinuous_b200 as kb
    rng = np.random.default_rng(7)
    n = 9
    fr = []
    for k in range(n):
        d = frames[k][0].copy()
        d[rng.random(d.shape) < 0.04] = 0                       # holes that move from frame to frame
        fr.append((d, frames[k][1]))
    pd = [torch.from_numpy(f[0].view(np.int16)).pin_memory() for f in fr]
    pc = [torch.from_numpy(f[1]).pin_memory() for f in fr]
    dd = [t.cuda() for t in pd]; dc = [t.cuda() for t in pc]
    cfg = dict(vol=256, odometry=odometry, voxel_shift=4)
    ref = kb.Tracker(kb.Config.default(**cfg))
    hinted = kb.Tracker(kb.Config.default(**cfg))             # hint before every frame, the first included, host pointers
    mixed = kb.Tracker(kb.Config.default(**cfg))              # hint before some frames only, device pointers
    skip = {3, 6}
    hinted.prefetch_frame(pd[0].data_ptr(), pc[0].data_ptr())
    for k in range(n):
        pa = ref.process_frame(fr[k][0], fr[k][1], k)
        pb = hinted.process_frame(pd[k].data_ptr(), pc[k].data_ptr(), k)
        pm = mixed.process_frame_device(dd[k], dc[k], k)
        if k + 1 < n:
            hinted.prefetch_frame(pd[k + 1].data_ptr(), pc[k + 1].data_ptr())
            if (k + 1) not in skip:
                mixed.prefetch_frame(dd[k + 1], dc[k + 1])
        for p in (pb, pm):
            assert list(pa.t) == list(p.t) and list(pa.R) == list(p.R) and list(pa.voxel_wrap) == list(p.voxel_wrap), k
    # every buffer kt_download_map exposes that the mode writes.  -r ray-casts one level, and builds no depth pyramid, maps or colour
    # inputs (Q10): those buffers are never written, and the depth pyramid and colour inputs never zeroed either.
    if odometry == 1:
        taps = [(which, 0) for which in (2, 3, 5, 6)]
    else:
        taps = [(which, level) for which in range(5) for level in range(4)] + [(which, 0) for which in (5, 6, 7, 8)]
    ta, ca = ref.export_volume()
    for trk in (hinted, mixed):
        tb, cb = trk.export_volume()
        assert (ta == tb).all() and (ca == cb).all()
        for which, level in taps:
            assert np.array_equal(ref.download_map(which, level), trk.download_map(which, level), equal_nan=True), (which, level)
        trk.close()
    ref.close()


_IDX64_SCRIPT = r"""
import hashlib, sys
import numpy as np
import kintinuous_b200 as kb
from kintinuous_b200 import synth
trk = kb.Tracker(kb.Config.default(vol=256, odometry=0, voxel_shift=2))
h = hashlib.sha256()
for k in range(8):
    d, c = synth.render(k)
    p = trk.process_frame(d, c, k)
    R, t, gc, w = p.as_tuple()
    h.update(np.ascontiguousarray(R).tobytes()); h.update(np.ascontiguousarray(t).tobytes()); h.update(np.ascontiguousarray(w).tobytes())
ts, cs = trk.export_volume()
h.update(ts.tobytes()); h.update(cs.tobytes())
for w_ in (2, 3, 5):
    h.update(np.ascontiguousarray(trk.download_map(w_, 0)).tobytes())
print("HASH", h.hexdigest())
"""


def test_kernel_variants_are_bit_identical(built):
    """Template instances that the default configuration does not take must give bit-identical trackers:
    * KT_FORCE_IDX64: 64-bit voxel indices in integrate and raycast (what the 2048^3 volume of BASELINE config 5 needs; the reference
      cannot run there, its int index overflows -- SURVEY.md D5), here on a 256^3 volume;
    * KT_INT_PREP=0: the colour update with the reference's per-voxel arithmetic (the operator-level golden tests pin that form against
      the reference) versus the default, which prepares the per-pixel colour weight and float RGB once per frame;
    * KT_INT_ZU=1: one voxel per step at 6 CTAs/SM (the default for volumes >= 1024^3);
    * KT_INT_NOBOX=1: integrate launched over the whole volume instead of the frustum's box of storage tiles (kt_frustum.hpp);
    * KT_ICP_STAGE_PASSES=2: a two-pass shared-memory stage, so that ICP level 0 streams its remaining passes from global memory as
      1280x960 does on one H100 (kt_icp.cu), versus the full stage;
    * KT_INT_SEQ_REPLAY=1: the running sums of a column replayed one float addition at a time up to its first voxel, as the reference
      does, versus the default exact fast-forward (kt_replay.cuh, replay_add)."""
    import subprocess
    import sys
    from conftest import ROOT
    out = {}
    for tag, extra in (("default", {}), ("idx64", {"KT_FORCE_IDX64": "1"}), ("noprep", {"KT_INT_PREP": "0"}), ("zu1", {"KT_INT_ZU": "1"}), ("seqreplay", {"KT_INT_SEQ_REPLAY": "1"}), ("nobox", {"KT_INT_NOBOX": "1"}), ("stage2", {"KT_ICP_STAGE_PASSES": "2"}),
                       ("idx64_noprep", {"KT_FORCE_IDX64": "1", "KT_INT_PREP": "0"})):
        env = dict(os.environ, PYTHONPATH=ROOT, **extra)
        r = subprocess.run([sys.executable, "-c", _IDX64_SCRIPT], env=env, capture_output=True, text=True, timeout=600, cwd=ROOT)
        assert r.returncode == 0, r.stderr[-2000:]
        out[tag] = [l for l in r.stdout.splitlines() if l.startswith("HASH")][0]
    assert len(set(out.values())) == 1, out


def test_config5_1280x960_into_2048(built):
    """BASELINE config 5 on one GPU: 1280x960 frames into a 2048^3 volume (51.5 GB, 2.9 mm voxels).  No reference exists at this size,
    so the check is against the synthetic scene's ground truth: the tracked pose follows the generator's trajectory and the model
    depth map raycast out of the volume reproduces the input depth to about a voxel."""
    import torch
    import kintinuous_b200 as kb
    from kintinuous_b200 import synth
    free, _ = torch.cuda.mem_get_info()
    if free < 70e9:
        pytest.skip("needs 70 GB of free device memory")
    rows, cols, V = 960, 1280, 2048
    trk = kb.Tracker(kb.Config.default(rows=rows, cols=cols, vol=V, odometry=0))
    voxel = 6.0 / V
    for k in range(4):
        d, c = synth.render(k, cols, rows)
        p = trk.process_frame(d, c, k)
        R, t, gc, w = p.as_tuple()
        Rg, tg = synth.pose(k)
        assert np.abs(t - (tg + 3.0)).max() < 2e-3, (k, t, tg)
        assert rot_angle(R, Rg.astype(np.float32)) < 1e-3, k
    vm = trk.download_map(2, 0).reshape(3, rows, cols)                # model vertex map (volume frame) raycast at the last pose
    zc = (vm - t.reshape(3, 1, 1))                                    # rotate into the camera: z_cam = R^T (v - t)
    z = np.einsum("i,ihw->hw", R[:, 2].astype(np.float64), zc.astype(np.float64))
    ok = np.isfinite(vm[0]) & (d > 0)
    assert ok.mean() > 0.9
    err = np.abs(z[ok] - d[ok] / 1000.0)
    assert np.median(err) < 1.0 * voxel, np.median(err)
    assert np.quantile(err, 0.95) < 4 * voxel
    trk.close()


def test_dense_pose_graph_and_pose_log(built, tmp_path):
    """KintinuousTracker::densePoseGraph / latestDensePoseId (KintinuousTracker.h:151-172, .cpp:529-536, :901-909) and the <saveFile>.poses
    trajectory outputPose appends per tracked frame (.cpp:199-218, :911-914): one DensePose per frame ([R | currentGlobalCamera], loop flag
    on the first), one text line per frame after the first, formatted as the reference streams it."""
    import kintinuous_b200 as kb
    from kintinuous_b200 import synth
    rows, cols = 120, 160
    log = str(tmp_path / "run.klg.poses")
    trk = kb.Tracker(kb.Config.default(rows=rows, cols=cols, vol=128, odometry=0, voxel_shift=2))
    trk.set_pose_log(log)
    poses = []
    for k in range(12):
        d, c = synth.render(k, cols, rows)
        p = trk.process_frame(d, c, 1000000 + 33333 * k)
        poses.append(p.as_tuple())
    assert trk.num_dense_poses() == 12
    for k in range(12):
        ts, M, loop = trk.dense_pose(k)
        R, t, g, w = poses[k]
        assert ts == 1000000 + 33333 * k and loop == (k == 0)
        assert np.array_equal(M[:3, :3], R) and np.array_equal(M[3], np.array([0, 0, 0, 1], np.float32))
        if k > 0:
            assert np.array_equal(M[:3, 3], g)                      # currentGlobalCamera of that frame (.cpp:581-596), before any shift of it
    trk.set_pose_log(None)
    lines = open(log).read().splitlines()
    assert len(lines) == 11                                         # no line for the first frame (.cpp:529-557 returns before outputPose)
    from scipy.spatial.transform import Rotation
    for k, line in enumerate(lines, start=1):
        f = line.split()
        R, t, g, w = poses[k]
        assert f[0] == "%.6f" % ((1000000 + 33333 * k) / 1000000.0)
        assert f[1:4] == ["%g" % float(v) for v in g]
        q = Rotation.from_matrix(R.astype(np.float64)).as_quat()
        got = np.array([float(x) for x in f[4:]])
        if np.dot(q, got) < 0:
            q = -q
        assert np.abs(got - q).max() < 2e-5
    trk.reset()
    assert trk.num_dense_poses() == 0
    trk.close()
